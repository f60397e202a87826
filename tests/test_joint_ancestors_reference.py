"""CPU suite: tests/joint_ancestors_reference.py, the reference of tests/test_gpu_joint_ancestors.py, and the reference
binary's joint reconstruction fixtures.

The max-product recursion attains the maximum over every assignment, enumerated in long double on trees of at most three
internal nodes; the reference binary's states are the restatement's wherever the restatement's decisions are not near
ties, and attain its optimum where they differ; and each plausible kernel bug of MUTATIONS changes a state or the joint
log-likelihood on a workload of the GPU file."""
import numpy as np
import pytest

from tests import batch_reference as br
from tests import joint_ancestors_reference as jr
from tests import test_gpu_joint_ancestors as G
from tests.test_gpu_batch_shapes import make_case, make_tree, partition

LD = br.LD


def _args(case, s, expm, col=None):
    return (case.w.tree, expm, case.V[s], case.W[s] if case.mix else None, case.branch_k,
            case.w.leaf_states[:, case.pats[s]] if col is None else col, case.w.ambig, case.root)


def enumerate_best(args):
    """max over every assignment of the internal nodes of the log joint probability, by brute force: a long-double array
    over all D^I assignments (every internal node resolved)."""
    tree, expm, V, W, branch_k, col, ambig, root = args
    L, I, D = tree.n_leaves, tree.n_internal, len(root)
    P = br.set_P(expm, V, W, branch_k)
    amb = np.asarray(ambig, dtype=LD)

    def axis(i, v):
        shape = [1] * I
        shape[i] = D
        return np.asarray(v, dtype=LD).reshape(shape)
    prob = axis(I - 1, root)
    for i, ch in enumerate(tree.children()):
        for c in ch:
            if c >= L:
                shape = [1] * I
                shape[i], shape[c - L] = D, D
                prob = prob * P[c].reshape(shape)
            elif col[c] >= 0:
                prob = prob * axis(i, P[c][:, col[c]])
            elif not jr.unresolved_leaf(col[c], amb):
                prob = prob * axis(i, (P[c] * amb[-col[c] - 1][None, :]).max(axis=1))
    with np.errstate(divide="ignore"):
        return np.log(prob.max())


SMALL = [(33, [[0, 0], [0, 0, 0]], False), (48, [[0, 0], 0, 0], True), (64, [0, [0, 0], 0], False)]


@pytest.mark.parametrize("D,spec,mix", SMALL, ids=["33", "48-mix", "64"])
def test_recursion_attains_enumerated_maximum(D, spec, mix):
    tmpl = br.compact_template(D, True, seed=3)
    w = partition(tmpl, make_tree(spec, seed=D), 40, seed=D, amb_frac=0.3)
    case = make_case(tmpl, w, 3, mix, seed=D)
    expm = br.ExpmCache(case.tmpl, br.expm_ld)
    amb_cols = np.nonzero((w.leaf_states < 0).any(axis=0))[0]
    assert len(amb_cols)
    for s, p in enumerate([int(amb_cols[0]), int(amb_cols[-1]), 0]):
        col = w.leaf_states[:, p].copy()
        if s == 2:
            col[0] = -1                               # a gap leaf
        args = _args(case, s, expm, col)
        states, l_star, _ = jr.joint_states(*args)
        assert np.all(states >= 0)
        assert abs(float(jr.assignment_lnl(*args, states) - l_star)) <= 1e-17 * abs(float(l_star))
        assert abs(float(enumerate_best(args) - l_star)) <= 1e-15 * abs(float(l_star)), (s, p)


def test_gaps_are_unresolved():
    """The GPU file's gap columns: every node -1 and l* = 0 for an all-gap column, -1 at a gapped cherry only."""
    case, expm, cols = G.gap_joint_case()
    cherry, _ = G.leaf_cherry(case.w.tree)
    states, l_star, _ = jr.joint_states(*_args(case, 0, expm, cols[0]))
    assert np.all(states == -1) and l_star == 0.0
    states, _, _ = jr.joint_states(*_args(case, 1, expm, cols[1]))
    assert states[cherry] == -1 and (states >= 0).sum() == case.w.tree.n_internal - 1
    states, _, _ = jr.joint_states(*_args(case, 2, expm, cols[2]))
    assert np.all(states >= 0)


@pytest.mark.parametrize("name", list(G.FIXTURES))
def test_fixture_agrees_with_restatement(name):
    w, g, V, W, branch_k = G.load_fixture(name)
    ex = G.CodonExpm(w, True)
    first = np.array([np.nonzero(w.site_to_pattern == p)[0][0] for p in range(w.S)])
    n_exact = 0
    for p in range(w.S):
        args = (w.tree, ex, V, W, branch_k, w.leaf_states[:, p], w.ambig, w.pi)
        states, l_star, margin = jr.joint_states(*args)
        got = g["states"][first[p]]
        assert np.array_equal(got < 0, states < 0), p
        if margin >= G.MARGIN:
            assert np.array_equal(got, states), p
            n_exact += 1
        else:
            assert abs(float(jr.assignment_lnl(*args, got) - l_star)) <= G.TOL, p
    assert n_exact >= w.S // 2


# ---------------------------------------------------------------------------------------------------------------------
# mutations: each plausible kernel bug changes a state or the joint log-likelihood on a GPU file's workload
# ---------------------------------------------------------------------------------------------------------------------
def _sweep(D, reversible, mix):
    def case():
        c, ex = G.sweep_joint_case(D, reversible, mix)
        return [_args(c, s, ex) for s in range(c.n)]
    return case


def _gaps():
    def case():
        c, ex, cols = G.gap_joint_case()
        return [_args(c, s, ex, cols[s]) for s in range(len(cols))]
    return case


def _ties():
    def case():
        c, ex, cols = G.tie_joint_case()
        return [_args(c, 0, ex, col) for col in cols]
    return case


MUTATION_CASES = {                  # mutation: a workload of tests/test_gpu_joint_ancestors.py
    "sum": _sweep(48, True, False),
    "ties_high": _ties(),
    "resolved_max": _sweep(33, True, False),
    "gap_resolved": _gaps(),
    "root_no_pi": _sweep(61, True, False),
    "own_argmax": _sweep(64, False, False),
    "component0": _sweep(48, False, True),
    "unresolved_state": _gaps(),
}


def test_every_mutation_has_a_case():
    assert set(MUTATION_CASES) == set(jr.MUTATIONS)


@pytest.mark.parametrize("mutation", list(MUTATION_CASES))
def test_mutation_changes_a_state_or_the_optimum(mutation):
    moved = 0
    for args in MUTATION_CASES[mutation]():
        st, ls, _ = jr.joint_states(*args)
        st2, ls2, _ = jr.joint_states(*args, mutate=(mutation,))
        if not np.array_equal(st, st2) or np.isinf(ls) != np.isinf(ls2) or (np.isfinite(ls) and abs(float(ls2 - ls)) > 10 * G.TOL):
            moved += 1
    print(f"{mutation}: {moved} sets changed")
    assert moved > 0, mutation
