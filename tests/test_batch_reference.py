"""CPU suite: tests/batch_reference.py, the reference of tests/test_gpu_batch_shapes.py.

The long-double exponential holds against mpmath at 30 digits and scipy, the long-double pruning against the oracle on
every tree shape, the compact templates against a direct construction, the columns of a 3-leaf star sum to 1, and --
what makes the GPU tests able to see a kernel bug at all -- each plausible bug of MUTATIONS, restated on the reference,
moves a set of the GPU file's own workloads by more than the tolerance that file holds the engine to."""
import math

import mpmath
import numpy as np
import pytest
import scipy.linalg

from hyphy_b200 import synth
from oracle import port
from tests import batch_reference as br
from tests import test_gpu_batch_shapes as G
from tests.test_gpu_shapes import TREES


def _site_lnl(sl, ss):
    return np.log(sl) - 64.0 * np.log(2.0) * ss


@pytest.mark.parametrize("D,length", [(33, 0.3), (33, 40.0), (64, 12.0)])
def test_expm_ld_against_mpmath(D, length):
    """30 significant digits; the larger norms need 5 and 8 squarings."""
    t = br.compact_template(D, D == 33, seed=9)
    A = br.dense(t, br.row_values(t, length, 1.0, 2.0))
    P = br.expm_ld(br.dense(t, br.row_values(t, length, 1.0, 2.0), br.LD))
    with mpmath.workdps(30):
        ref = mpmath.expm(mpmath.matrix(A.tolist()))
        err = max(abs(ref[i, j] - mpmath.mpf(str(P[i, j]))) for i in range(D) for j in range(D))
    assert err <= 1e-15 * max(1.0, float(br.norm1(A))), (float(br.norm1(A)), float(err))


@pytest.mark.parametrize("reversible", [True, False])
@pytest.mark.parametrize("D", [33, 47, 48, 61, 64])
def test_expm_ld_against_scipy(D, reversible):
    t = br.compact_template(D, reversible, seed=1)
    for length in (1e-8, 0.05, 0.7, 6.0, 30.0):
        A = br.dense(t, br.row_values(t, length, 0.8, 3.0))
        P = br.expm_ld(br.dense(t, br.row_values(t, length, 0.8, 3.0), br.LD))
        np.testing.assert_allclose(P.astype(np.float64), scipy.linalg.expm(A), rtol=0, atol=1e-14, err_msg=f"t={length}")
        assert np.abs(P.sum(axis=1) - 1).max() <= 1e-15


@pytest.mark.parametrize("reversible", [True, False])
@pytest.mark.parametrize("D", [33, 48, 64])
def test_compact_template_matches_direct_construction(D, reversible):
    t = br.compact_template(D, reversible, seed=1)
    assert t.nF == 2 * D and len(t.ei) == 4 * D and len(set(t.ei)) == 4 * D
    v = np.random.default_rng(D).uniform(0.1, 2.0, t.nF)
    Q = np.zeros((D, D))
    c = D // 3
    for e, (a, b) in enumerate([(i, (i + 1) % D) for i in range(D)] + [(i, (i + c) % D) for i in range(D)]):
        if reversible:
            Q[a, b], Q[b, a] = v[e] * t.cf[b], v[e] * t.cf[a]
        else:
            Q[a, b], Q[b, a] = v[e % D], v[D + e % D]
    Q[np.diag_indices(D)] = -Q.sum(axis=1)
    np.testing.assert_allclose(br.dense(t, v), Q, rtol=1e-15, atol=0)
    flux = t.cf[:, None] * Q if reversible else Q
    off = ~np.eye(D, dtype=bool)
    if reversible:
        np.testing.assert_allclose(flux[off], flux.T[off], rtol=1e-14)
    else:
        assert np.abs(flux - flux.T)[off].max() > 0.1 * np.abs(flux[off]).max()
        P = br.expm_ld(br.dense(t, t.base * 0.5, br.LD))
        assert np.abs(P - P.T).max() > 1e-3                       # a transposed matrix is another matrix


@pytest.mark.parametrize("shape", list(TREES))
def test_prune_ld_against_oracle(shape):
    """One column per tree shape (with an ambiguity code) under the oracle's matrices: the long-double recursion against
    port.prune's scaled fp64 recursion."""
    tmpl = br.compact_template(61, True, seed=2)
    tree = G.make_tree(TREES[shape], seed=len(shape))
    w = G.partition(tmpl, tree, 30, seed=len(shape), amb_frac=0.1)
    P = np.stack([port.expm(br.dense(tmpl, br.row_values(tmpl, tree.t[b], 1.0, 1.5))) for b in range(tree.n_branches)])
    root = np.random.default_rng(3).dirichlet(np.full(61, 2.0))
    cols = w.leaf_states[:, :2].T
    w1 = synth.Workload("one", tree, 61, root, w.Q_classes, w.class_weights, cols.T.copy(), w.ambig, np.ones(2, np.int64), np.arange(2))
    sl, ss = port.prune(w1, P)
    want = _site_lnl(sl, ss)
    got = br.prune_ld(tree, P, cols, w.ambig, root).astype(np.float64)
    np.testing.assert_allclose(got, want, rtol=1e-13)


@pytest.mark.parametrize("mix", [False, True])
def test_star3_columns_sum_to_one(mix):
    D = 33
    case = G.star3_case(D, mix)
    P = br.set_P(br.ExpmCache(case.tmpl, br.expm_ld), case.V[0], None if case.W is None else case.W[0], case.branch_k)
    lnl = br.prune_ld(case.w.tree, P, G.all_columns(D), case.w.ambig, case.root)
    assert len(lnl) == D ** 3
    assert abs(np.exp(lnl).sum() - 1) <= 1e-15                   # root vector and weights sum to 1 in fp64


# ---------------------------------------------------------------------------------------------------------------------
# mutations: each plausible kernel bug moves a workload of the GPU file beyond that file's tolerance
# ---------------------------------------------------------------------------------------------------------------------
MUTATION_CASES = {                  # mutation: (the GPU file's case, patterns or columns, its tolerance)
    "drop_last": (lambda: G.sweep_case(48, True, True), "patterns", "sweep"),
    "w0_all": (lambda: G.sweep_case(48, True, True), "patterns", "sweep"),
    "transpose": (lambda: G.sweep_case(48, False, False), "patterns", "sweep"),
    "amb_off_by_one": (lambda: G.sweep_case(48, True, False), "columns", "sweep"),
    "pad_leak": (lambda: G.sweep_case(48, True, False), "columns", "sweep"),
    "no_wide_rescale": (lambda: G.shape_case("star400", 61, True), "patterns", "shapes"),
}


def test_every_mutation_has_a_case():
    assert set(MUTATION_CASES) == set(br.MUTATIONS)


def _shift(make, what, mutation):
    """Largest relative change of a set's log-likelihood under the mutation (None: none), on the GPU file's workload."""
    case = make()
    expm = G.expm_for(case)
    ref = np.asarray(G.reference(case, expm, what), np.float64)
    mut = np.asarray(G.reference(case, expm, what, mutate=() if mutation is None else (mutation,)), np.float64)
    with np.errstate(invalid="ignore"):
        err = np.abs(mut - ref) / np.abs(ref)
    return float(np.where(np.isnan(err), np.inf, err).max())


@pytest.mark.parametrize("mutation", list(MUTATION_CASES))
def test_mutation_moves_a_set_beyond_tolerance(mutation):
    make, what, tol_key = MUTATION_CASES[mutation]
    assert _shift(make, what, None) == 0.0                       # unmutated, nothing moves: the check below has teeth
    shift = _shift(make, what, mutation)
    print(f"{mutation}: largest relative shift {shift:.2e} against tolerance {G.TOL[tol_key]:.0e}")
    assert shift > 10 * G.TOL[tol_key] or math.isinf(shift), (mutation, shift)
