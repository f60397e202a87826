"""CPU suite for tests/site_rates_reference.py, the reference of hb2_batch_site_rates: it agrees with the oracle's fp64
exponential and pruning, rate 0 gives identity matrices, and every restated kernel bug moves the GPU file's workloads
beyond its tolerances."""
import numpy as np
import pytest

from oracle import port
from tests import batch_reference as br
from tests import site_rates_reference as sr
from tests.test_gpu_site_rates import SWEEP_TREE, TOL, rate_workload, rate_sets, reference, rel_err


@pytest.mark.parametrize("D,reversible", [(3, True), (4, True), (20, True), (7, False)])
@pytest.mark.parametrize("r", [0.05, 1.0, 7.0])
def test_reference_agrees_with_oracle(D, reversible, r):
    t, w, _ = rate_workload(SWEEP_TREE, D, seed=11, reversible=reversible)
    A = w.Qt()[0]
    got = sr.site_lnl(w.tree, A, r, w.leaf_states.T, w.ambig, w.pi)
    P = np.stack([port.expm(r * Ab, False) for Ab in A])
    sl, ss = port.prune(w, P)
    ref = np.log(sl) - 64.0 * np.log(2.0) * ss
    assert float(np.max(np.abs(np.asarray(got, np.float64) - ref) / np.abs(ref))) <= 1e-12


@pytest.mark.parametrize("D", [2, 5, 17, 32])
def test_small_template_is_a_rate_matrix(D):
    for reversible in (True, False):
        t = sr.small_template(D, reversible)
        Q = br.dense(t, t.base)
        assert np.allclose(Q.sum(axis=1), 0.0, atol=1e-14)
        assert np.all(Q[~np.eye(D, dtype=bool)] >= 0) and np.all(np.diag(Q) < 0)
        pi = t.cf if reversible else np.full(D, 1.0 / D)
        assert abs(-(pi * np.diag(Q)).sum() - 1.0) <= 1e-13
        if reversible:
            assert np.allclose(pi[:, None] * Q, (pi[:, None] * Q).T, atol=1e-14)


def test_rate_zero_gives_identity():
    t, w, root = rate_workload(SWEEP_TREE, 5, seed=12)
    P = sr.rate_P(w.Qt()[0], 0.0, w.tree.n_leaves, sr.RateExpm())
    assert np.array_equal(P, np.broadcast_to(np.eye(5, dtype=br.LD), P.shape))


@pytest.mark.parametrize("mutation", sorted(sr.MUTATIONS))
def test_each_mutation_is_caught(mutation):
    """Every restated bug moves the sweep workload (5 states padded to 8, ambiguity rows, a non-uniform root) by far more
    than the GPU file's tolerance."""
    t, w, root = rate_workload(SWEEP_TREE, 5, seed=1)
    pats, rates = rate_sets(w, seed=5)
    clean = reference(w, root, pats, rates)
    bad = reference(w, root, pats, rates, mutate={mutation})
    with np.errstate(invalid="ignore"):
        err = np.nan_to_num(rel_err(bad, clean), nan=np.inf)
    assert float(err.max()) > 1e3 * max(TOL.values()), (mutation, float(err.max()))
