"""GPU suite (pytest -m gpu): hb2_simulate against its numpy restatement (tests/simulate_reference.py) fed the engine's own
transition matrices, bit for bit; stream properties; the distribution of simulated data against exact probabilities; no
effect on evaluations; a round trip through a new likelihood function; refusals."""
import ctypes as C

import numpy as np
import pytest

from hyphy_b200 import synth, engine, LikelihoodFunction, Partition
from oracle import port
from tests import handover_cases as hc
from tests import simulate_reference as ref
from tests.test_gpu_shapes import flat_tree, star, polytomy, caterpillar
from tests.test_simulate_reference import pattern_probabilities, pooled_chisquare

pytestmark = pytest.mark.gpu

FLAGS = {"fp64": engine.FLAG_FORCE_FP64, "tc": engine.FLAG_DEFAULT}
RATES = np.array([0.5, 1.0, 1.6, 2.4])                  # class rate multipliers
WEIGHTS4 = np.array([0.2, 0.0, 0.5, 0.3])               # class 1 is never drawn: its matrices are never handed over


@pytest.fixture(scope="module", autouse=True)
def _need_gpu(engine_lib):
    assert engine.device_count() > 0, "GPU tests need a CUDA device (no fallback exists)"


def template(D):
    if D == 61:
        return hc.gy94_template(), hc.gy94_rates(2.0, 0.4)
    return hc.gtr_template(D, 100 + D)


def make_partition(tree, D, n_classes, mode="fp64", n_sites=64, seed=0):
    rng = np.random.default_rng(seed)
    ls = rng.integers(0, D, size=(tree.n_leaves, n_sites))
    return Partition(n_sites, D, tree.n_leaves, tree.n_internal, n_classes, tree.flat_parents, ls, None,
                     np.ones(n_sites, dtype=np.int64), flags=FLAGS[mode])


def hand_over(part, tree, D, kind, classes):
    """Matrices of every branch for the listed classes: dense rate, dense transition, compiled or two-component mixture."""
    tm, x = template(D)
    nb = tree.n_branches
    nodes = np.arange(nb)
    t = tree.t[:nb]
    if kind == "compiled":
        tm.define(part, 0)
    for c in classes:
        r = RATES[c]
        if kind == "rate":
            part.set_matrices(c, nodes, np.stack([tm.Q(x) * (r * tb) for tb in t]), engine.MATRIX_RATE)
        elif kind == "trans":
            part.set_matrices(c, nodes, np.stack([port.expm(tm.Q(x) * (r * tb)) for tb in t]), engine.MATRIX_TRANS)
        elif kind == "compiled":
            part.set_matrices_compiled(c, nodes, np.stack([x * (r * tb) for tb in t]))
        else:
            M = np.stack([np.stack([tm.Q(x) * (r * tb * om) for om in (0.3, 2.0)]) for tb in t])
            part.set_mixture_matrices(c, nodes, M, np.tile([0.7, 0.3], (nb, 1)))


def engine_P(part, classes):
    """The engine's transition matrices [C, B, D, D] (zero for classes not listed)."""
    P = np.zeros((part.C, part.B, part.D, part.D))
    for c in classes:
        for b in range(part.B):
            P[c, b] = part.read_transition(c, b)
    return P


def root_freqs(D, seed=5):
    return np.random.default_rng(seed).dirichlet(np.full(D, 3.0))


def check_exact(part, tree, classes, weights, pi, n, seed, first=0):
    leaf, nodes, cls = part.simulate(n, pi, weights, seed, first, want_nodes=True, want_classes=True)
    rl, rn, rc = ref.simulate(engine_P(part, classes), weights, pi, tree.flat_parents, tree.n_leaves, n, seed, first)
    assert np.array_equal(cls, rc)
    assert np.array_equal(nodes, rn)
    assert np.array_equal(leaf, rl)
    return leaf, nodes, cls


# ---------------------------------------------------------------------------------------------------------------------
# bit-exact against the reference
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_classes", [1, 4])
@pytest.mark.parametrize("kind", ["rate", "trans", "compiled", "mixture"])
@pytest.mark.parametrize("D,mode", [(4, "fp64"), (20, "fp64"), (61, "fp64"), (61, "tc")])
def test_matches_reference(D, mode, kind, n_classes):
    tree = synth.random_tree(12, 40 + D, mean_t=0.15)
    part = make_partition(tree, D, n_classes, mode)
    classes = [0] if n_classes == 1 else [0, 2, 3]
    hand_over(part, tree, D, kind, classes)
    weights = None if n_classes == 1 else WEIGHTS4
    _, _, cls = check_exact(part, tree, classes, weights, root_freqs(D), 3000, seed=0x1234_5678_9ABC + D)
    if n_classes == 4:
        assert set(np.unique(cls)) == {0, 2, 3}
    part.close()


@pytest.mark.parametrize("D", [4, 20])
@pytest.mark.parametrize("shape", ["star40", "poly7", "caterpillar700"])
def test_tree_shapes_match_reference(shape, D):
    """A star (one internal node), a polytomy, and a caterpillar whose internal states do not fit in shared memory."""
    tree = flat_tree({"star40": star(40), "poly7": polytomy(7), "caterpillar700": caterpillar(700)}[shape], mean_t=0.1, seed=3)
    part = make_partition(tree, D, 2)
    hand_over(part, tree, D, "rate", [0, 1])
    check_exact(part, tree, [0, 1], np.array([1.0, 3.0]), root_freqs(D), 2000, seed=77)
    part.close()


@pytest.mark.parametrize("n_classes", [65, 70, 130])
def test_many_classes_match_reference(n_classes):
    """More than 64 rate classes: the class draw searches the whole weight vector.  Class 64 has weight 0 and receives
    no matrices, so a draw that stopped at index 64 would read rows that were never built."""
    tree = synth.random_tree(6, 17, mean_t=0.2)
    part = make_partition(tree, 4, n_classes)
    rng = np.random.default_rng(n_classes)
    w = rng.random(n_classes)
    w[64] = 0.0
    w[rng.integers(0, 64, 3)] = 0.0
    if n_classes > 65:
        w[-1] = 0.0
    active = [c for c in range(n_classes) if w[c] > 0]
    tm, x = template(4)
    nodes = np.arange(tree.n_branches)
    for c in active:
        r = 0.2 + 0.05 * c
        part.set_matrices(c, nodes, np.stack([port.expm(tm.Q(x) * (r * tb)) for tb in tree.t[:tree.n_branches]]), engine.MATRIX_TRANS)
    _, _, cls = check_exact(part, tree, active, w, root_freqs(4), 20000, seed=123)
    assert 64 not in set(cls) and set(cls) <= set(active)
    if n_classes > 65:
        assert (cls > 64).any()
    part.close()


# ---------------------------------------------------------------------------------------------------------------------
# stream properties
# ---------------------------------------------------------------------------------------------------------------------
def test_split_calls_seeds_and_chunks():
    tree = synth.random_tree(9, 11, mean_t=0.2)
    part = make_partition(tree, 4, 4)
    hand_over(part, tree, 4, "rate", [0, 2, 3])
    pi = root_freqs(4)
    n = 300_000                                             # more than one chunk of 2^18 sites
    whole = check_exact(part, tree, [0, 2, 3], WEIGHTS4, pi, n, seed=42)
    h = n // 2
    a = part.simulate(h, pi, WEIGHTS4, 42, 0, True, True)
    b = part.simulate(n - h, pi, WEIGHTS4, 42, h, True, True)
    for x, y, z in zip(whole, a, b):
        assert np.array_equal(x, np.concatenate([y, z], axis=-1))
    other = part.simulate(n, pi, WEIGHTS4, 43)[0]
    assert (other != whole[0]).mean() > 0.3
    empty = part.simulate(0, pi, WEIGHTS4, 42, 0, True, True)
    assert empty[0].shape == (9, 0) and empty[1].shape == (7, 0) and empty[2].shape == (0,)
    part.close()


# ---------------------------------------------------------------------------------------------------------------------
# distribution
# ---------------------------------------------------------------------------------------------------------------------
def test_pattern_distribution_five_leaves_two_classes():
    tree = synth.random_tree(5, 8, mean_t=0.3)
    part = make_partition(tree, 4, 2)
    hand_over(part, tree, 4, "rate", [0, 1])
    w = np.array([0.35, 0.65])
    pi = root_freqs(4, 9)
    n = 1 << 22
    leaf, _, _ = part.simulate(n, pi, w, seed=20261017)
    P = engine_P(part, [0, 1])
    prob = sum(w[c] * pattern_probabilities(tree, P[c], pi) for c in range(2))
    assert abs(prob.sum() - 1.0) < 1e-12
    code = np.zeros(n, dtype=np.int64)
    for l in range(5):
        code = code * 4 + leaf[l]
    counts = np.bincount(code, minlength=1024)
    assert pooled_chisquare(counts, n * prob) > 1e-4
    part.close()


def test_codon_leaf_marginals():
    tree = synth.random_tree(6, 21, mean_t=0.4)
    part = make_partition(tree, 61, 1, "tc")
    hand_over(part, tree, 61, "compiled", [0])
    pi = synth.codon_frequencies(synth.DEFAULT_POSFREQ)
    n = 400_000
    leaf, _, _ = part.simulate(n, pi, None, seed=3)
    P = engine_P(part, [0])[0]
    L, fp = tree.n_leaves, tree.flat_parents
    for l in range(L):
        path = [l]
        while fp[path[-1]] != tree.n_internal - 1:
            path.append(L + fp[path[-1]])
        M = np.eye(61)
        for node in reversed(path):                     # root -> leaf
            M = M @ P[node]
        p = pooled_chisquare(np.bincount(leaf[l], minlength=61), n * (pi @ M))
        assert p > 1e-4, (l, p)
    part.close()


# ---------------------------------------------------------------------------------------------------------------------
# no interference with evaluations
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D,mode", [(4, "fp64"), (61, "fp64"), (61, "tc")])
def test_evaluations_unchanged(D, mode):
    w = hc.workload(D, 14, 300, 4)
    tree = w.tree
    lf = LikelihoodFunction(w, flags=FLAGS[mode])
    hand_over(lf.part, tree, D, "compiled", range(4))
    before = lf.compute(want_sites=True)
    lf.simulate(5000, seed=1, want_nodes=True, want_classes=True)
    after = lf.compute(want_sites=True)
    assert before[0] == after[0]
    assert np.array_equal(before[1], after[1]) and np.array_equal(before[2], after[2])
    node = 3
    # the branch cache built before a simulation gives the same values after it
    lf.part.branch_cache_build(node, w.pi)
    bc1 = lf.part.branch_cache_evaluate(w.class_weights, want_sites=True)
    lf.simulate(5000, seed=2)
    bc2 = lf.part.branch_cache_evaluate(w.class_weights, want_sites=True)
    assert bc1[0] == bc2[0] and np.array_equal(bc1[1], bc2[1]) and np.array_equal(bc1[2], bc2[2])
    lf.close()


# ---------------------------------------------------------------------------------------------------------------------
# round trip
# ---------------------------------------------------------------------------------------------------------------------
def test_round_trip_through_a_new_likelihood_function():
    w = synth.codon_workload(10, 60, 4)
    lf = LikelihoodFunction(w)
    lf.set_all_matrices()
    leaf, _, _ = lf.simulate(20_000, seed=11)
    lf.close()
    ls, freq, s2p = synth.compress(leaf)
    assert freq.sum() == 20_000
    w2 = synth.Workload("simulated", w.tree, 61, w.pi, w.Q_classes, w.class_weights, ls, np.zeros((0, 61)), freq, s2p, None, w.meta)
    ref_lnl, _ = port.lnl(w2)
    for flags, rtol in ((engine.FLAG_DEFAULT, 1e-7), (engine.FLAG_FORCE_FP64, 1e-10)):
        lf2 = LikelihoodFunction(w2, flags=flags)
        lf2.set_all_matrices()
        got = lf2.compute()
        lf2.close()
        assert abs(got - ref_lnl) <= rtol * abs(ref_lnl), (flags, got, ref_lnl)


# ---------------------------------------------------------------------------------------------------------------------
# refusals
# ---------------------------------------------------------------------------------------------------------------------
def raw_simulate(part, weights, pi, n, seed=0, first=0):
    """hb2_simulate on sentinel-filled outputs of max(n, 1) sites; returns (rc, leaf, nodes, classes)."""
    m = max(n, 1)
    leaf = np.full((part.L, m), -7, dtype=np.int64)
    nodes = np.full((part.I, m), -7, dtype=np.int64)
    cls = np.full(m, -7, dtype=np.int32)
    pw = None if weights is None else np.ascontiguousarray(weights, dtype=np.float64).ctypes.data_as(C.POINTER(C.c_double))
    keep = (weights, np.ascontiguousarray(pi, dtype=np.float64))
    rc = part._lib.hb2_simulate(part._h, pw, keep[1].ctypes.data_as(C.POINTER(C.c_double)), n, seed, first,
                                leaf.ctypes.data_as(C.POINTER(C.c_int64)), nodes.ctypes.data_as(C.POINTER(C.c_int64)),
                                cls.ctypes.data_as(C.POINTER(C.c_int32)))
    return rc, leaf, nodes, cls


def assert_refused(part, weights, pi, n=100, match="", first=0):
    rc, leaf, nodes, cls = raw_simulate(part, weights, pi, n, first=first)
    assert rc != 0
    msg = engine.load_library().hb2_last_error().decode()
    assert match in msg, msg
    assert (leaf == -7).all() and (nodes == -7).all() and (cls == -7).all()
    return msg


def test_refusals():
    tree = synth.random_tree(7, 5)
    part = make_partition(tree, 4, 2)
    hand_over(part, tree, 4, "rate", [0])                   # class 1 never receives a matrix
    pi = root_freqs(4)
    w = np.array([1.0, 0.0])
    assert raw_simulate(part, w, pi, 100)[0] == 0           # the valid call the refusals below deviate from
    assert_refused(part, w, pi, n=-1, match="negative")
    assert_refused(part, w, pi, first=-5, match="firstSite")
    for bad in ([-1.0, 2.0], [np.nan, 1.0], [0.0, 0.0], [np.inf, 1.0]):
        assert_refused(part, np.array(bad), pi, match="class weights")
    for bad in ([0.5, -0.1, 0.3, 0.3], [np.nan, 1, 1, 1], [0.0, 0.0, 0.0, 0.0]):
        assert_refused(part, w, np.array(bad), match="root frequencies")
    assert_refused(part, None, pi, match="weights may be null")
    assert_refused(part, np.array([1.0, 1.0]), pi, match="rate class 1, node 0")
    # a transition matrix with a row that sums to zero, and one with a NaN total, in a drawn class
    P = np.stack([port.expm(hc.gtr_template(4, 104)[0].Q(hc.gtr_template(4, 104)[1]) * tb) for tb in tree.t[:tree.n_branches]])
    P[4, 2] = 0.0
    part.set_matrices(0, np.arange(tree.n_branches), P, engine.MATRIX_TRANS)
    assert_refused(part, w, pi, match="row 2 of the transition matrix of rate class 0, node 4")
    P[4, 2] = 0.25
    P[6, 1, 3] = np.inf
    part.set_matrices(0, np.arange(tree.n_branches), P, engine.MATRIX_TRANS)
    assert_refused(part, w, pi, match="row 1 of the transition matrix of rate class 0, node 6")
    # the same matrices in a class that is never drawn are not looked at
    P[6, 1, 3] = 0.0
    part.set_matrices(0, np.arange(tree.n_branches), P, engine.MATRIX_TRANS)
    P[0, 0] = np.nan
    part.set_matrices(1, np.arange(tree.n_branches), P, engine.MATRIX_TRANS)
    assert raw_simulate(part, w, pi, 100)[0] == 0
    assert_refused(part, np.array([1.0, 1.0]), pi, match="row 0 of the transition matrix of rate class 1, node 0")
    part.close()
