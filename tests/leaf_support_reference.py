"""Plain high-precision reference of hb2_batch_leaf_support (leaf state imputation: ReconstructAncestors(MARGINAL,
DOLEAVES), as MEME and PRIME run it per site with --impute-states): for every leaf, the distribution of its state given
every other leaf of one set's column.

  * brute_support: what the reference does (likefunc2.cpp:974-1006 and :1083-1093) -- for every (leaf l, state k), the
    column with l's code replaced by k, pruned by batch_reference.prune_ld, and each leaf's D values normalised;
  * outside_support: the kernel's algorithm restated in long double without scaling -- one inside pass, one pre-order
    pass of outside vectors with sibling products without division (branch_rows_reference.outside_rows' structure), and
    for each leaf l: u[k] = sum_p A_l[p] P_l[p][k], normalised.  It takes `mutate`, a set of labels that each restate one
    plausible bug of that algorithm (MUTATIONS); the CPU suite shows that the unmutated form equals brute_support and
    that each bug moves an entry of the GPU file's workloads beyond its tolerances.

Both return [L, D] long-double rows; a row whose total is 0 or not finite is NaN in every entry.  Sets are given as for
batch_reference.set_P: rows V [R, nF], weights W [R] or None (one row per branch), branch_k [B].  `expm` is a
batch_reference.ExpmCache (long-double or oracle exponentials).  No test functions live here."""
import numpy as np

from tests import batch_reference as br

LD = br.LD

MUTATIONS = {
    "posterior": "the leaf's own observation is multiplied in (the posterior given all the data, not the predictive)",
    "leaf_through_P": "the leaf product goes through P (u[k] = sum_p A[p] P[k][p]) instead of its column",
    "leaf_component0": "the leaf product goes through its branch's first component instead of its mixture",
    "outside_no_siblings": "the leaf's A is its parent's outside vector without the sibling messages",
    "sibling_self": "the sibling product also includes the leaf's own message",
    "root_ones": "the root's outside vector is all ones instead of the root frequencies",
    "drop_third_child": "the third child of a wide node is left out of its siblings' products",
}


def offsets(branch_k):
    return np.concatenate([[0], np.cumsum(branch_k)]).astype(np.int64)


def normalise(u):
    """Rows u [.., D] divided by their totals; NaN rows where a total is 0 or not finite."""
    u = np.asarray(u, dtype=LD)
    tot = u.sum(axis=-1, keepdims=True)
    ok = np.isfinite(tot) & (tot != 0)
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.where(ok, u / np.where(ok, tot, 1), LD(np.nan))


def forced_columns(col, D):
    """[L * D, L]: the column with leaf l's code replaced by k, row l * D + k."""
    col = np.asarray(col, dtype=np.int64)
    L = len(col)
    out = np.repeat(col[None, :], L * D, axis=0)
    for l in range(L):
        out[l * D:(l + 1) * D, l] = np.arange(D)
    return out


def brute_support(tree, expm, V, W, branch_k, col, ambig, root):
    """[L, D]: the reference's procedure, every forced column pruned in long double and normalised per leaf."""
    P = br.set_P(expm, V, W, branch_k)
    D, L = P.shape[-1], tree.n_leaves
    with np.errstate(divide="ignore"):
        lnl = np.asarray(br.prune_ld(tree, P, forced_columns(col, D), ambig, root), dtype=LD).reshape(L, D)
    with np.errstate(invalid="ignore"):
        return normalise(np.exp(lnl))


def outside_support(tree, expm, V, W, branch_k, col, ambig, root, mutate=()):
    """[L, D] by one inside and one outside pass (the kernel's order, no scaling)."""
    L, D = tree.n_leaves, len(root)
    P = br.set_P(expm, V, W, branch_k)
    off = offsets(branch_k)
    amb = np.asarray(ambig, dtype=LD)
    kids = tree.children()
    inside = [None] * (L + tree.n_internal)
    for c in range(L):
        code = col[c]
        if code >= 0:
            inside[c] = np.zeros(D, dtype=LD)
            inside[c][code] = 1
        else:
            inside[c] = amb[-code - 1].copy()
    msg = [None] * len(inside)
    for i, ch in enumerate(kids):
        v = np.ones(D, dtype=LD)
        for c in ch:
            msg[c] = P[c] @ inside[c]
            v = v * msg[c]
        inside[L + i] = v
    root0 = np.ones(D, dtype=LD) if "root_ones" in mutate else np.asarray(root, dtype=LD)
    outside = {L + tree.n_internal - 1: root0}
    out = np.empty((L, D), dtype=LD)
    for i in reversed(range(tree.n_internal)):
        ch = kids[i]
        for c in ch:
            A = outside[L + i].copy()
            if not (c < L and "outside_no_siblings" in mutate):
                for q, c2 in enumerate(ch):
                    if c2 == c and "sibling_self" not in mutate:
                        continue
                    if q == 2 and "drop_third_child" in mutate:
                        continue
                    A = A * msg[c2]
            if c >= L:
                outside[c] = A @ P[c]
                continue
            Pc = expm(V[off[c]]) if "leaf_component0" in mutate else P[c]
            u = Pc @ A if "leaf_through_P" in mutate else A @ Pc
            if "posterior" in mutate:
                u = u * inside[c]
            out[c] = u
    return normalise(out)
