"""CPU suite: the numpy restatement of hb2_simulate's stream (tests/simulate_reference.py) -- Philox4x32-10 known answers,
the edges of the draw rule, and the distribution of simulated patterns against exact pattern probabilities."""
import itertools

import numpy as np
import scipy.stats

from hyphy_b200 import synth
from oracle import port
from tests import simulate_reference as ref


def _words(hexes):
    return np.array([int(h, 16) for h in hexes.split()], dtype=np.uint64)


def test_philox_known_answers():
    """Random123's known-answer vectors for philox4x32_10."""
    cases = [("00000000 00000000 00000000 00000000", "00000000 00000000", "6627e8d5 e169c58d bc57ac4c 9b00dbd8"),
             ("ffffffff ffffffff ffffffff ffffffff", "ffffffff ffffffff", "408f276d 41c83b0e a20bc7c6 6d5451fd"),
             ("243f6a88 85a308d3 13198a2e 03707344", "a4093822 299f31d0", "d16cfe09 94fdcceb 5001e420 24126ea1")]
    for ctr, key, out in cases:
        got = ref.philox4x32_10(_words(ctr), _words(key))
        assert [f"{int(x):08x}" for x in got] == out.split()


def test_uniform_uses_53_bits():
    u = ref.uniforms(np.arange(100000), 3, 12345)
    assert u.min() >= 0.0 and u.max() < 1.0
    k = u * 2.0 ** 53
    assert np.array_equal(k, np.floor(k))                 # multiples of 2^-53
    assert abs(u.mean() - 0.5) < 0.005


def test_draw_rule_skips_entries_that_are_not_positive():
    v = np.array([0.0, -1.0, np.nan, 2.0, 0.0, 1.0, -0.0])
    c, last = ref.prefix(v)
    assert last == 5
    assert list(c) == [0.0, 0.0, 0.0, 2.0, 2.0, 3.0, 3.0]
    u = np.array([0.0, 0.5, 0.6666, 2.0 / 3.0, 0.9999999])
    got = ref.draw(np.broadcast_to(c, (len(u), len(v))), np.full(len(u), last), u)
    # t = u * 3: [0, 1.5, 1.9998, 2, 2.9999997] -> first j with t < c_j
    assert list(got) == [3, 3, 3, 5, 5]


def test_draw_rule_falls_back_to_last_positive_entry():
    """u * T rounding up to T finds no j with t < c_j: the last positive entry is drawn, never a trailing zero.  For u < 1
    that takes a total at the bottom of the normal range or below, where the product's rounding step is coarse."""
    tiny = 5e-324                                         # 2^-1074
    v = np.array([tiny, 0.0, 2 * tiny, 0.0, 0.0])
    c, last = ref.prefix(v)
    assert last == 2 and c[-1] == 3 * tiny
    u = np.array([1.0 - 2.0 ** -53, 0.9, 0.1])
    assert u[0] * c[-1] == c[-1] and u[1] * c[-1] == c[-1]
    assert list(ref.draw(np.broadcast_to(c, (3, 5)), np.full(3, last), u)) == [2, 2, 0]
    # an entry absorbed by rounding still counts as positive for the fall-back
    c2, last2 = ref.prefix(np.array([1.0, 1e-17, 0.0]))
    assert c2[0] == c2[1] and last2 == 1
    # with a normal total, u * T < T for every u < 1: the fall-back is never reached
    T = np.array([1.0, 1.25, 2.0 - 2.0 ** -52, 3.0e300])
    assert np.all((1.0 - 2.0 ** -53) * T < T)


def test_draw_frequencies_follow_the_weights():
    v = np.array([0.1, 0.0, 0.6, 0.3])
    c, last = ref.prefix(v)
    n = 200000
    u = ref.uniforms(np.arange(n), 0, 7)
    got = ref.draw(np.broadcast_to(c, (n, 4)), np.full(n, last), u)
    counts = np.bincount(got, minlength=4)
    assert counts[1] == 0
    p = scipy.stats.chisquare(counts[[0, 2, 3]], n * v[[0, 2, 3]]).pvalue
    assert p > 1e-4


def pattern_probabilities(tree, P, pi):
    """Exact probability of every leaf pattern of a small tree, by the oracle's pruning (one pattern per column)."""
    L, D = tree.n_leaves, P.shape[-1]
    pats = np.array(list(itertools.product(range(D), repeat=L)), dtype=np.int64).T      # [L, D^L], leaf 0 slowest
    w = synth.Workload("patterns", tree, D, pi, [np.zeros((D, D))], np.array([1.0]), pats, np.zeros((0, D)),
                       np.ones(pats.shape[1], dtype=np.int64), np.arange(pats.shape[1]))
    sl, ss = port.prune(w, P)
    return sl * 2.0 ** (-64.0 * ss)


def pooled_chisquare(observed, expected, min_expected=5.0):
    """Pearson chi-square with the cells of expected count < min_expected pooled into one."""
    small = expected < min_expected
    obs = np.append(observed[~small], observed[small].sum())
    exp = np.append(expected[~small], expected[small].sum())
    if exp[-1] == 0:
        obs, exp = obs[:-1], exp[:-1]
    return scipy.stats.chisquare(obs, exp * obs.sum() / exp.sum()).pvalue


def test_reference_pattern_distribution_on_three_leaves():
    tree = synth.FlatTree(3, 1, np.array([0, 0, 0, -1]), ["a", "b", "c", "r"], np.array([0.1, 0.3, 0.7, 0.0]), "")
    pi = np.array([0.1, 0.2, 0.3, 0.4])
    Q = synth.hky85_Q(3.0, pi)
    P = np.stack([synth._expm_np(Q * t) for t in tree.t[:3]])
    n = 200000
    leaf, nodes, cls = ref.simulate(P[None], None, pi, tree.flat_parents, 3, n, seed=2026)
    assert leaf.shape == (3, n) and nodes.shape == (1, n) and not cls.any()
    prob = pattern_probabilities(tree, P, pi)
    assert abs(prob.sum() - 1.0) < 1e-12
    counts = np.bincount(leaf[0] * 16 + leaf[1] * 4 + leaf[2], minlength=64)
    assert pooled_chisquare(counts, n * prob) > 1e-4
    assert pooled_chisquare(np.bincount(nodes[0], minlength=4), n * pi) > 1e-4


def test_reference_sites_depend_on_the_global_site_only():
    tree = synth.random_tree(6, 3)
    rng = np.random.default_rng(1)
    P = rng.random((2, tree.n_branches, 5, 5))
    a = ref.simulate(P, [0.3, 0.7], np.ones(5), tree.flat_parents, 6, 1000, seed=9)
    b = ref.simulate(P, [0.3, 0.7], np.ones(5), tree.flat_parents, 6, 400, seed=9, first_site=600)
    for x, y in zip(a, b):
        assert np.array_equal(x[..., 600:], y)
    c = ref.simulate(P, [0.3, 0.7], np.ones(5), tree.flat_parents, 6, 1000, seed=10)
    assert not np.array_equal(a[0], c[0])
