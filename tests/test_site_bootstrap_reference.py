"""CPU suite: the numpy restatement of hb2_batch_site_simulate's stream (tests/site_bootstrap_reference.py) -- set 0 is
hb2_simulate's stream, the set word changes the draws, splitting is invisible, and simulated columns follow exact pattern
probabilities."""
import numpy as np

from hyphy_b200 import synth
from tests import simulate_reference as sim_ref
from tests import site_bootstrap_reference as ref
from tests.test_simulate_reference import pattern_probabilities, pooled_chisquare


def _tree4():
    """((a,b),(c,d)) in flat post-order: leaves 0..3, internal nodes 4 (a,b), 5 (c,d), root 6."""
    return synth.FlatTree(4, 3, np.array([0, 0, 1, 1, 2, 2, -1]), ["a", "b", "c", "d", "ab", "cd", "r"],
                          np.array([0.1, 0.3, 0.2, 0.5, 0.15, 0.25, 0.0]), "")


def test_set_zero_is_the_simulate_stream():
    """t = 0 with one set reproduces hb2_simulate's reference for one class on the same matrices, bit for bit."""
    tree = synth.random_tree(7, 3)
    rng = np.random.default_rng(3)
    P = rng.random((tree.n_branches, 6, 6))
    pi = rng.random(6)
    leaf, nodes = ref.simulate_sets(P[None], pi, tree.flat_parents, 7, 500, seed=77, first_rep=1000)
    sl, sn, _ = sim_ref.simulate(P[None], None, pi, tree.flat_parents, 7, 500, seed=77, first_site=1000)
    assert leaf.shape == (1, 500, 7) and nodes.shape == (1, 500, tree.n_internal)
    assert np.array_equal(leaf[0], sl.T)
    assert np.array_equal(nodes[0], sn.T)


def test_set_word_changes_the_draws():
    tree = synth.random_tree(6, 4)
    rng = np.random.default_rng(4)
    P = np.broadcast_to(rng.random((tree.n_branches, 5, 5)), (2, tree.n_branches, 5, 5))
    leaf, _ = ref.simulate_sets(P, np.ones(5), tree.flat_parents, 6, 300, seed=5)
    assert not np.array_equal(leaf[0], leaf[1])
    # a set's columns depend on its global set and replicate only
    one, _ = ref.simulate_sets(P[1:], np.ones(5), tree.flat_parents, 6, 100, seed=5, first_set=1, first_rep=200)
    assert np.array_equal(one[0], leaf[1, 200:])


def test_columns_follow_pattern_probabilities():
    """Column-pattern frequencies on a 4-leaf, 4-state tree against exact probabilities (chi-square)."""
    tree = _tree4()
    pi = np.array([0.1, 0.2, 0.3, 0.4])
    Q = synth.hky85_Q(2.5, pi)
    P = np.stack([synth._expm_np(Q * t) for t in tree.t[:tree.n_branches]])
    n = 200000
    leaf, nodes = ref.simulate_sets(P[None], pi, tree.flat_parents, 4, n, seed=2027, first_set=12)
    prob = pattern_probabilities(tree, P, pi)
    assert abs(prob.sum() - 1.0) < 1e-12
    code = ((leaf[0, :, 0] * 4 + leaf[0, :, 1]) * 4 + leaf[0, :, 2]) * 4 + leaf[0, :, 3]
    assert pooled_chisquare(np.bincount(code, minlength=256), n * prob) > 1e-4
    assert pooled_chisquare(np.bincount(nodes[0, :, -1], minlength=4), n * pi) > 1e-4


def test_mixture_rows_in_component_order():
    rng = np.random.default_rng(6)
    P = rng.random((5, 3, 3))
    w = rng.random(5)
    got = ref.mix(P, w, [2, 1, 2])
    assert np.array_equal(got[1], w[2] * P[2])
    assert np.array_equal(got[2], w[3] * P[3] + w[4] * P[4])
