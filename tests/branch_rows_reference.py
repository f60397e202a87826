"""Plain high-precision reference of hb2_batch_branch_component_likelihoods (MEME's branch-level empirical Bayes,
MEME.bf:886-944): the log-likelihood of one set with one branch pinned to one of its mixture components.

  * brute_rows: what MEME itself does -- for every (branch, component) row, the set's matrices (batch_reference.set_P)
    with that branch's matrix replaced by the row's exponential alone, pruned by batch_reference.prune_ld;
  * outside_rows: the kernel's algorithm restated in long double without scaling -- one inside pass, one pre-order pass
    of outside vectors, sibling products without division, each row scored as A_b . (P_r in_c).  It takes `mutate`, a set
    of labels that each restate one plausible bug of that algorithm (MUTATIONS); the CPU suite shows that the unmutated
    form equals brute_rows and that each bug moves the GPU file's workloads beyond its tolerances.

`expm` is a batch_reference.ExpmCache (long-double or oracle exponentials).  No test functions live here."""
import numpy as np

from tests import batch_reference as br

LD = br.LD

MUTATIONS = {
    "outside_through_P": "the outside vector goes through P (O_c[j] = sum_p A[p] P[j][p]) instead of its transpose",
    "sibling_self": "the sibling product also includes the branch's own message",
    "root_ones": "the root's outside vector is all ones instead of the root frequencies",
    "row_mixed": "a row is scored with the branch's mixed matrix instead of its own component",
    "drop_third_child": "the third child of a wide node is left out of its siblings' products",
    "root_stationary": "the root's outside vector is the template's stationary vector instead of the caller's root vector",
    "message_transposed": "the outside pass's child messages go through the transpose (m_c = P^T in_c)",
    "outside_component0": "an internal child's outside vector goes through its branch's first component, not its mixture",
}


def _row_offsets(branch_k):
    return np.concatenate([[0], np.cumsum(branch_k)]).astype(np.int64)


def brute_rows(tree, expm, V, W, branch_k, col, ambig, root):
    """[R] long-double log-likelihoods of column `col` [L]: row r of branch b pins b to Exp(V[r]) with weight 1."""
    P = br.set_P(expm, V, W, branch_k)
    off = _row_offsets(branch_k)
    out = np.empty(off[-1], dtype=LD)
    for b in range(len(branch_k)):
        for r in range(off[b], off[b + 1]):
            Pr = P.copy()
            Pr[b] = expm(V[r])
            out[r] = br.prune_ld(tree, Pr, col[None, :], ambig, root)[0]
    return out


def site_ld(tree, expm, V, W, branch_k, col, ambig, root):
    """The set's own mixed log-likelihood (long double)."""
    return br.prune_ld(tree, br.set_P(expm, V, W, branch_k), col[None, :], ambig, root)[0]


def stationary(t):
    """The stationary vector of a batch_reference.Template at its base rates: the column frequencies where it has them
    (pi_i q_ij is symmetric for every alpha, beta), else the left null vector of its rate matrix."""
    if t.cf is not None:
        return np.asarray(t.cf, dtype=LD)
    Q = br.dense(t, t.base)
    vt = np.linalg.svd(Q.T)[2]
    pi = np.abs(vt[-1])
    return np.asarray(pi / pi.sum(), dtype=LD)


def outside_rows(tree, expm, V, W, branch_k, col, ambig, root, mutate=()):
    """[R] long-double log-likelihoods by one inside and one outside pass (the kernel's order, no scaling).  The
    'root_stationary' mutation reads the template of `expm` (a batch_reference.ExpmCache)."""
    L, D = tree.n_leaves, len(root)
    P = br.set_P(expm, V, W, branch_k)
    off = _row_offsets(branch_k)
    amb = np.asarray(ambig, dtype=LD)
    kids = tree.children()
    inside = [None] * (L + tree.n_internal)                      # subtree vector of every flat node
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
    side_msg = msg
    if "message_transposed" in mutate:                           # the inside pass stays right; the outside pass's copy not
        side_msg = [None if m is None else P[c].T @ inside[c] for c, m in enumerate(msg)]
    out = np.empty(off[-1], dtype=LD)
    root0 = np.asarray(root, dtype=LD)
    if "root_ones" in mutate:
        root0 = np.ones(D, dtype=LD)
    elif "root_stationary" in mutate:
        root0 = stationary(expm.t)
    outside = {L + tree.n_internal - 1: root0}
    for i in reversed(range(tree.n_internal)):
        ch = kids[i]
        for pos, c in enumerate(ch):
            A = outside[L + i].copy()
            for q, c2 in enumerate(ch):
                if c2 == c and "sibling_self" not in mutate:
                    continue
                if q == 2 and "drop_third_child" in mutate:
                    continue
                A = A * side_msg[c2]
            for r in range(off[c], off[c + 1]):
                Pr = P[c] if "row_mixed" in mutate else expm(V[r])
                out[r] = np.log(A @ (Pr @ inside[c]))
            if c >= L:
                Pc = expm(V[off[c]]) if "outside_component0" in mutate else P[c]
                outside[c] = Pc @ A if "outside_through_P" in mutate else A @ Pc
    return out
