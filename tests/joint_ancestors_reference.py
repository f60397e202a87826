"""Plain high-precision reference of hb2_batch_joint_ancestors (the joint maximum-likelihood reconstruction of
ReconstructAncestors, as FEL, MEME and PRIME run it per site through ancestral.build): Pupko's max-product recursion of
the reference's RecoverAncestralSequences (tree.cpp:4209-4510), restated in long double without scaling.

  1. children in increasing flat id, each parent vector starting at 1;
  2. a resolved leaf in state a multiplies its parent by P[p][a], with no max;
  3. an ambiguous leaf or an internal child with vector x multiplies it by max_c P[p][c] x[c], the scan over ascending c
     by strict > against a running maximum that starts at 0 with index 0 (ties to the lowest c; 0 and NaN never win);
  4. an unresolved child (a leaf whose row is 1 in all D states, or an internal node all of whose children are
     unresolved) takes state -1 and does not multiply its parent;
  5. no rescaling is needed in long double;
  6. the root state is argmax_c pi_c J_root[c] by the same rule, -1 for every node when the root is unresolved;
  7. traceback: each internal node takes its argument at its parent's state, -1 below a -1.

joint_states returns (states [I], l_star, margin): l_star the natural log of pi_r J_root[r] (0.0 for an unresolved root,
-inf for a product of 0), margin the smallest relative gap between the best and the second-best product at any decision
on the chosen path (1.0 when no decision has a second candidate).  assignment_lnl gives the log joint probability of any
assignment under the same conventions (unresolved parts contribute nothing, an ambiguous leaf its best state).  It takes
`mutate`, a set of labels that each restate one plausible kernel bug (MUTATIONS).  Sets are given as for
batch_reference.set_P.  No test functions live here."""
import numpy as np

from tests import batch_reference as br

LD = br.LD

MUTATIONS = {
    "sum": "a child's factor is the sum over its states instead of the max",
    "ties_high": "ties go to the highest index (>= instead of > in the scan)",
    "resolved_max": "a resolved leaf takes the max over its matrix row instead of P[p][code]",
    "gap_resolved": "a leaf whose row is all ones is treated as resolved: it multiplies its parent by its max",
    "root_no_pi": "the root state is the argmax of J_root without the root vector",
    "own_argmax": "a child's state is the argmax of its own vector instead of its parent's row of the table",
    "component0": "a branch's matrix is its mixture's first component instead of the mixture",
    "unresolved_state": "an internal node all of whose children are unresolved is given a state (its vector is all ones)",
}


def _scan(vals, high=False):
    """(best, index, second) of the reference's strict-> scan from 0 with index 0 over vals; `high` sends ties to the
    highest index."""
    best, idx, second = LD(0), 0, LD(0)
    for c, t in enumerate(vals):
        if t > best or (high and t == best and t > 0):
            second, best, idx = best, t, c
        elif t > second:
            second = t
    return best, idx, second


def set_matrices(expm, V, W, branch_k, mutate=()):
    if "component0" in mutate and W is not None:
        off = np.concatenate([[0], np.cumsum(branch_k)]).astype(np.int64)
        return np.stack([expm(V[off[b]]) for b in range(len(branch_k))])
    return br.set_P(expm, V, W, branch_k)


def unresolved_leaf(code, amb):
    return code < 0 and bool(np.all(amb[-code - 1] != 0))


def joint_states(tree, expm, V, W, branch_k, col, ambig, root, mutate=()):
    L, I, D = tree.n_leaves, tree.n_internal, len(root)
    P = set_matrices(expm, V, W, branch_k, mutate)
    amb = np.asarray(ambig, dtype=LD)
    high = "ties_high" in mutate
    kids = tree.children()
    J = [None] * I
    unres = [False] * I
    arg, gap = {}, {}                      # internal child index -> [D] argument / relative margin per parent state
    for i, ch in enumerate(kids):
        v = np.ones(D, dtype=LD)
        open_ = True
        for c in ch:
            Pc = P[c]
            if c < L:
                code = int(col[c])
                if code >= 0:
                    f = np.array([_scan(Pc[p])[0] for p in range(D)]) if "resolved_max" in mutate else Pc[:, code]
                else:
                    if unresolved_leaf(code, amb) and "gap_resolved" not in mutate:
                        continue
                    x = amb[-code - 1]
                    f = (Pc * x[None, :]).sum(axis=1) if "sum" in mutate else \
                        np.array([_scan(Pc[p] * x, high)[0] for p in range(D)])
            else:
                ci = c - L
                if unres[ci] and "unresolved_state" not in mutate:
                    continue
                x = J[ci]
                f = np.empty(D, dtype=LD)
                a = np.zeros(D, dtype=np.int64)
                g = np.ones(D, dtype=LD)
                for p in range(D):
                    prod = Pc[p] * x
                    best, a[p], second = _scan(prod, high)
                    f[p] = prod.sum() if "sum" in mutate else best
                    g[p] = (best - second) / best if best > 0 else LD(0)
                arg[ci], gap[ci] = a, g
            v = v * f
            open_ = False
        J[i] = v
        unres[i] = open_
    states = np.full(I, -1, dtype=np.int64)
    if unres[I - 1]:
        return states, LD(0), 1.0
    x = J[I - 1] if "root_no_pi" in mutate else J[I - 1] * np.asarray(root, dtype=LD)
    best, r, second = _scan(x, high)
    margin = float((best - second) / best) if best > 0 else 0.0
    states[I - 1] = r
    for i in reversed(range(I)):
        for c in kids[i]:
            if c < L:
                continue
            ci = c - L
            if (unres[ci] and "unresolved_state" not in mutate) or states[i] < 0:
                continue
            if "own_argmax" in mutate:
                states[ci] = _scan(J[ci])[1]
            else:
                states[ci] = arg[ci][states[i]]
                margin = min(margin, float(gap[ci][states[i]]))
    with np.errstate(divide="ignore"):
        l_star = np.log(LD(x[r]))
    return states, l_star, margin


def assignment_lnl(tree, expm, V, W, branch_k, col, ambig, root, states):
    """Long-double log joint probability of internal states [I] (-1: unresolved): pi at the root, P[s_parent][s_child] on
    every branch between resolved internal nodes, P[s][code] for a resolved leaf, the max over an ambiguous leaf's nonzero
    states, nothing for unresolved leaves and subtrees; 0.0 when the root is -1."""
    L, I = tree.n_leaves, tree.n_internal
    P = br.set_P(expm, V, W, branch_k)
    amb = np.asarray(ambig, dtype=LD)
    if states[I - 1] < 0:
        return LD(0)
    prob = LD(np.asarray(root, dtype=LD)[states[I - 1]])
    for i, ch in enumerate(tree.children()):
        s = states[i]
        if s < 0:
            continue
        for c in ch:
            if c >= L:
                if states[c - L] >= 0:
                    prob = prob * P[c][s, states[c - L]]
                continue
            code = int(col[c])
            if code >= 0:
                prob = prob * P[c][s, code]
            elif not unresolved_leaf(code, amb):
                prob = prob * _scan(P[c][s] * amb[-code - 1])[0]
    with np.errstate(divide="ignore"):
        return np.log(prob)
