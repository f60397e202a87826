"""CPU suite: the oracle on the shapes of tests/test_gpu_shapes.py, where no output of the reference binary pins it.

The oracle (oracle/hb2_oracle.c) is pinned to the reference binary on the fixtures of tests/golden/ only.  Here it is held to
independent plain implementations: scipy.linalg.expm for the transition matrices, and a numpy.longdouble Felsenstein
recursion without any scaling (tests.test_gpu_shapes.longdouble_sites) for the likelihoods, on odd state counts, star,
polytomy and caterpillar trees, a single pattern, and the stars whose products underflow a double."""
import numpy as np
import pytest
import scipy.linalg

from hyphy_b200 import synth
from oracle import port
from tests.test_gpu_shapes import (TREES, UNDERFLOW, flat_tree, inject_ambiguity, log2_unscaled_max, longdouble_sites,
                                   oracle_P, tree_workload, underflow_workload, edge_matrices, _site_lnl)

# Per-pattern agreement.  Both sides use the same matrices, so what differs is the rounding of the products: under 1e-16
# relative per operation in fp64, about 2^-64 in the long-double recursion, a few hundred operations per pattern on the
# largest trees here.
SITE_ATOL = 1e-12


def test_longdouble_has_the_exponent_range():
    assert np.finfo(np.longdouble).minexp < -10000


def _check_sites(w, P):
    sl, ss = port.prune(w, P)
    np.testing.assert_allclose(_site_lnl(sl, ss), longdouble_sites(w, P), rtol=0, atol=SITE_ATOL)


@pytest.mark.parametrize("D", [3, 5, 7, 9, 17, 33, 63, 64])
def test_oracle_odd_state_counts_random_tree(D):
    w = tree_workload(synth.random_tree(14, 2, mean_t=0.3), D, 200, seed=3)
    inject_ambiguity(w, np.random.default_rng(D))
    _check_sites(w, oracle_P(w))


@pytest.mark.parametrize("D", [3, 7, 9, 33, 64])
def test_oracle_expm_against_scipy(D):
    """The oracle's exp(Qt) at the lengths test_gpu_shapes.py uses, against scipy, with the tolerances used there for the
    engine's matrices (the oracle agrees to better than a third of them)."""
    Q, _ = synth.gtr_like_Q(D, 5 + D)
    for label, A, atol in edge_matrices(Q):
        P = port.expm(A, False)
        if label == "zero":
            np.testing.assert_array_equal(P, np.eye(D))
            continue
        np.testing.assert_allclose(P, scipy.linalg.expm(A), rtol=0, atol=atol / 3, err_msg=label)


@pytest.mark.parametrize("D", [4, 9, 61])
@pytest.mark.parametrize("shape", ["star3", "star40", "star400", "poly7", "poly33", "all_internal", "bifurcating_root",
                                   "caterpillar700", "leaf_by_deep"])
def test_oracle_tree_shapes(shape, D):
    w = tree_workload(flat_tree(TREES[shape], mean_t=0.2, seed=len(shape)), D, 150, seed=9)
    _check_sites(w, oracle_P(w))


@pytest.mark.parametrize("D", [2, 7, 20, 64])
def test_oracle_one_pattern(D):
    w = tree_workload(synth.random_tree(10, 4, mean_t=0.3), D, 50, seed=2, n_patterns=1)
    assert w.S == 1
    _check_sites(w, oracle_P(w))


@pytest.mark.parametrize("name", list(UNDERFLOW))
def test_oracle_underflow_stars(name):
    """Where the product over the children leaves the double range, the oracle's 2^64 boosts keep it exact -- up to the
    reference's cap of sqrt(DBL_MAX * 1e-10) ~ 2^495 per node (tree.cpp:129,182).  Below that, like the reference, it
    returns a likelihood of 0 (the 1500-leaf nucleotide star)."""
    w = underflow_workload(name)
    P = oracle_P(w)
    assert np.mean(log2_unscaled_max(w, P) < -1022) > 0.5
    sl, ss = port.prune(w, P)
    ref = longdouble_sites(w, P)
    assert np.all(np.isfinite(ref))
    if name == "nuc1500":
        assert np.mean(sl == 0.0) > 0.5
        ok = sl > 0
    else:
        ok = np.ones(w.S, dtype=bool)
        assert np.all(sl > 0)
    np.testing.assert_allclose(_site_lnl(sl[ok], ss[ok]), ref[ok], rtol=0, atol=SITE_ATOL)
