"""GPU suite (pytest -m gpu): hb2_batch_joint_ancestors, the joint maximum-likelihood states of every internal node
(ReconstructAncestors, FEL's, MEME's and PRIME's ancestral.build at every site), against the unmodified reference binary's
fixtures and the long-double restatement of its max-product recursion (tests/joint_ancestors_reference.py):

  1. the reference binary's states: bsrel_12x80_k3 (mixture layout, K = 3 on every branch), mg94_8x60_c1 (plain) and
     mg94_8x60_c1_gaps (plain, half the codons ambiguous or gaps);
  2. every state count 33..64 where the kernels change behaviour, reversible and not, plain sets and mixture sets with
     branchK taking 1..4 in one set, ambiguity rows;
  3. every tree shape of tests/test_gpu_shapes.py at 48 states, the 400-leaf star and the 700-leaf caterpillar included;
  4. the caller's root vector: Dirichlet, uniform, sparse (a zero state is never the root's), zeros (state 0, -inf);
  5. exact ties under identity matrices (zero formula values): the lowest compatible state, state 0 for disagreeing
     leaves, the lowest state of an intersection of partial ambiguities;
  6. gaps: an all-gap column, a gapped cherry, a single gap leaf;
  7. identities: plain sets = unit-weight mixtures, siteLnL = the likelihood entry points, fp64 = default partitions,
     all bit for bit;
  8. NaN weights and formula values confined to their set; chunks of more than 1024 sets; repeated calls;
  9. non-interference with evaluations, the branch cache and the other batch entry points' workspace; every refusal
     (class-group mode needs two ranks: tests/test_multigpu.py's territory, not exercised here).

The agreement rule, wherever states are compared: on every set whose long-double margin (the smallest relative gap
between the best and second-best product of a decision on the chosen path) is at least MARGIN the states are the
reference's exactly; on every set the long-double log probability of the engine's states and the engine's jointLnL are
within TOL of the optimum; -1 nodes always match."""
import dataclasses
import functools
import re

import numpy as np
import pytest

from hyphy_b200 import LikelihoodFunction, synth, engine
from hyphy_b200.engine import _check, _d, _i, _dp, _ip
from tests import golden_cases as gc
from tests import joint_ancestors_reference as jr
from tests.test_gpu_batch_mixture import LF, meme_sets
from tests.test_gpu_batch_shapes import SWEEP, new_lf
from tests.test_gpu_branch_rows import CodonExpm
from tests.test_gpu_leaf_support import fixture_sets, shape_support_case, sweep_support_case
from tests.test_gpu_shapes import TREES, flat_tree, star, tree_workload

pytestmark = pytest.mark.gpu

# |jointLnL - l*| and |log P(engine's states) - l*| in long double: ten times the largest error measured on one H100 80GB
# HBM3 (700 W), rounded up to a power of ten.  Measured: 1.1e-14 over the fixtures, sweep, root, tie, gap and small-tree
# cases; 4.1e-12 on the 400-leaf star and the 700-leaf caterpillar (LARGE_TOL, the trees of 100 branches or more, whose
# l* runs to thousands)
TOL = 1e-13
LARGE_TOL = 1e-10
MARGIN = 1e-10
FIXTURES = {"bsrel_12x80_k3": True, "mg94_8x60_c1": False, "mg94_8x60_c1_gaps": False}     # name: mixture layout
JOINT_CASES = {"mg94_8x60_c1_gaps": lambda: synth.codon_workload(8, 60, 1, ambig_frac=0.5)}    # tools/make_golden.py
_worst = [0.0]


@pytest.fixture(scope="module", autouse=True)
def _need_gpu(engine_lib):
    assert engine.device_count() > 0, "GPU tests need a CUDA device (no fallback exists)"
    yield
    print(f"[joint ancestors] largest error against l*: {_worst[0]:.2e}")


# ---------------------------------------------------------------------------------------------------------------------
# workloads, calls and references
# ---------------------------------------------------------------------------------------------------------------------
def load_fixture(name):
    """(workload, fixture, V, W, branch_k) of a _joint fixture; the workload is the one the binary saw."""
    w = JOINT_CASES[name]() if name in JOINT_CASES else gc.load(name)[0]
    g = np.load(gc.GOLDEN_DIR + f"/{name}_joint.npz")
    assert str(g["checksum"]) == gc.checksum(w)
    V, W, branch_k = fixture_sets(w)
    return w, g, V, W, branch_k


def sweep_joint_case(D, reversible, mix):
    return sweep_support_case(D, reversible, mix)


def leaf_cherry(tree):
    """(internal index, its two leaves) of the first internal node whose children are two leaves."""
    L = tree.n_leaves
    for i, ch in enumerate(tree.children()):
        if len(ch) == 2 and all(c < L for c in ch):
            return i, list(ch)
    raise AssertionError("no cherry")


def _with_columns(w, cols, ambig):
    """w with its first len(cols) patterns replaced by cols, every other ambiguous code by -1, and ambiguity rows ambig."""
    ls = w.leaf_states.copy()
    ls[ls < 0] = -1
    ls[:, :len(cols)] = np.asarray(cols).T
    return synth.Workload(w.name, w.tree, w.D, w.pi, w.Q_classes, w.class_weights, ls, np.asarray(ambig, np.float64),
                          w.pattern_freq, w.site_to_pattern, None, w.meta)


def _rows(D, *sets):
    a = np.zeros((len(sets), D))
    for r, s in enumerate(sets):
        a[r, list(s)] = 1.0
    return a


@functools.lru_cache(maxsize=None)
def gap_joint_case():
    """(case, expm, cols) on the 48-state sweep partition: an all-gap column, a gapped cherry, a single gap leaf."""
    case, expm = sweep_support_case(48, True, False)
    w = case.w
    L = w.tree.n_leaves
    _, leaves = leaf_cherry(w.tree)
    base = np.asarray(w.leaf_states[:, 0]).copy()
    base[base < 0] = 7
    cherry = base.copy()
    cherry[leaves] = -1
    one = base.copy()
    one[L - 1] = -1
    cols = [np.full(L, -1), cherry, one]
    w2 = _with_columns(w, cols, _rows(w.D, range(w.D), (3, 5, 9), (5, 9, 20)))
    case2 = dataclasses.replace(case, w=w2, pats=np.arange(case.n) % 3)
    return case2, expm, [np.asarray(c) for c in cols]


@functools.lru_cache(maxsize=None)
def tie_joint_case():
    """(case, expm, cols) on the 48-state sweep partition with zero formula values (every P the identity) and a uniform
    root: a constant column, every leaf {3,5,9}, disagreeing leaves, leaves {3,5,9} and {5,9,20} alternating."""
    case, expm = sweep_support_case(48, True, False)
    w = case.w
    L, D = w.tree.n_leaves, w.D
    alt = np.where(np.arange(L) % 2 == 0, -2, -3)
    dis = np.full(L, 7)
    dis[0] = 3
    cols = [np.full(L, 7), np.full(L, -2), dis, alt]
    w2 = _with_columns(w, cols, _rows(D, range(D), (3, 5, 9), (5, 9, 20)))
    V = np.zeros((len(cols),) + case.V.shape[1:])
    case2 = dataclasses.replace(case, w=w2, V=V, pats=np.arange(len(cols)), root=np.full(D, 1.0 / D), mid=case.mid[:len(cols)],
                                cols=case.cols[:len(cols)])
    return case2, expm, cols


def joint_call(lf, case, V=None, W=None, root=None, pats=None):
    """(states, jointLnL) of a batch-shapes Case; siteLnL checked against the likelihood entry point bit for bit."""
    V = case.V if V is None else V
    W = (case.W if case.mix else None) if W is None else W
    root = case.root if root is None else root
    pats = case.pats if pats is None else pats
    bk = case.branch_k if W is not None else None
    st, jl, site = lf.part.batch_joint_ancestors(pats, V, root, weights=W, branch_k=bk, want_site=True)
    if W is None:
        want = lf.part.batch_site_likelihoods(pats, V, root)
    else:
        want = lf.part.batch_site_mixture_likelihoods(pats, V, W, root, branch_k=bk)
    assert np.array_equal(site, want, equal_nan=True)
    st2, jl2 = lf.part.batch_joint_ancestors(pats, V, root, weights=W, branch_k=bk)
    assert np.array_equal(st, st2) and np.array_equal(jl, jl2, equal_nan=True)
    return st, jl


def check_agreement(st, jl, args_of, sets, label, want_states=None, tol=TOL):
    """The agreement rule over sets; args_of(s) gives joint_states' arguments of set s.  want_states: the reference
    binary's states instead of the restatement's."""
    worst, exact = 0.0, 0
    D = None
    for k, s in enumerate(sets):
        args = args_of(s)
        D = len(args[7])
        ref, l_star, margin = jr.joint_states(*args)
        want = ref if want_states is None else want_states[k]
        assert np.all((st[k] >= -1) & (st[k] < D)), (label, s)
        assert np.array_equal(st[k] < 0, want < 0), (label, s, st[k], want)
        if margin >= MARGIN:
            assert np.array_equal(st[k], want), (label, s, st[k], want, margin)
            exact += 1
        if np.isinf(l_star) or l_star == 0.0:
            assert jl[k] == l_star, (label, s, jl[k], l_star)
            continue
        e1 = abs(float(jr.assignment_lnl(*args, st[k]) - l_star))
        e2 = abs(float(jl[k] - l_star))
        worst = max(worst, e1, e2)
    _worst[0] = max(_worst[0], worst)
    print(f"[{label}] {len(sets)} sets, {exact} compared state by state; largest error against l*: {worst:.2e}")
    assert worst <= tol, (label, worst)
    return exact


def case_args(case, expm, cols=None, V=None, W=None, root=None):
    V = case.V if V is None else V
    W = (case.W if case.mix else None) if W is None else W
    root = case.root if root is None else root

    def args_of(s):
        col = case.w.leaf_states[:, case.pats[s]] if cols is None else cols[s]
        return (case.w.tree, expm, V[s], None if W is None else W[s], case.branch_k, col, case.w.ambig, root)
    return args_of


# ---------------------------------------------------------------------------------------------------------------------
# 1. the reference binary's states
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(FIXTURES))
def test_fixture_matches_reference(name):
    """Every pattern of the fixture (tools/make_golden.py --joint), one set per pattern."""
    w, g, V, W, branch_k = load_fixture(name)
    assert (W is not None) == FIXTURES[name]
    pats = np.arange(w.S)
    lf = LF(w)
    Vs = np.ascontiguousarray(np.broadcast_to(V, (w.S,) + V.shape))
    Ws = None if W is None else np.ascontiguousarray(np.broadcast_to(W, (w.S,) + W.shape))
    st, jl = lf.part.batch_joint_ancestors(pats, Vs, w.pi, weights=Ws, branch_k=None if W is None else branch_k)
    lf.close()
    first = np.array([np.nonzero(w.site_to_pattern == p)[0][0] for p in range(w.S)])
    ex = CodonExpm(w, True)
    exact = check_agreement(st, jl, lambda p: (w.tree, ex, V, W, branch_k, w.leaf_states[:, p], w.ambig, w.pi), pats,
                            f"fixture {name}", want_states=g["states"][first])
    assert exact >= w.S // 2
    assert np.array_equal(st[w.site_to_pattern] < 0, g["states"] < 0)


# ---------------------------------------------------------------------------------------------------------------------
# 2. state counts, 7. identities
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D,reversible", SWEEP, ids=[f"{d}{'' if r else '-nonrev'}" for d, r in SWEEP])
def test_state_sweep(D, reversible):
    for mix in (False, True):
        case, expm = sweep_joint_case(D, reversible, mix)
        if mix:
            assert set(case.branch_k) == {1, 2, 3, 4}
        assert (case.w.leaf_states[:, case.pats] < 0).any()
        out = {}
        for flags in (engine.FLAG_FORCE_FP64, engine.FLAG_DEFAULT):
            lf = new_lf(case, flags)
            out[flags] = joint_call(lf, case)
            lf.close()
        st, jl = out[engine.FLAG_FORCE_FP64]
        assert np.array_equal(st, out[engine.FLAG_DEFAULT][0]) and np.array_equal(jl, out[engine.FLAG_DEFAULT][1])
        check_agreement(st, jl, case_args(case, expm), range(case.n), f"sweep D={D} rev={reversible} mix={mix}")


@pytest.mark.parametrize("D,reversible", [(33, False), (61, True), (64, True)], ids=["33-nonrev", "61", "64"])
def test_plain_equals_unit_weight_mixture(D, reversible):
    case, _ = sweep_joint_case(D, reversible, False)
    lf = new_lf(case)
    st, jl = joint_call(lf, case)
    B = case.w.tree.n_branches
    st2, jl2 = lf.part.batch_joint_ancestors(case.pats, case.V, case.root, weights=np.ones((case.n, B)),
                                             branch_k=np.ones(B, np.int64))
    lf.close()
    assert np.array_equal(st, st2) and np.array_equal(jl, jl2)


# ---------------------------------------------------------------------------------------------------------------------
# 3. tree shapes
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", list(TREES))
def test_tree_shapes(shape):
    for mix in (False, True):
        case, expm = shape_support_case(shape, mix)
        lf = new_lf(case)
        st, jl = joint_call(lf, case)
        lf.close()
        big = case.w.tree.n_branches >= 100
        check_agreement(st, jl, case_args(case, expm), range(2) if big else range(case.n), f"shape {shape} mix={mix}",
                        tol=LARGE_TOL if big else TOL)


# ---------------------------------------------------------------------------------------------------------------------
# 4. the caller's root vector
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mix", [False, True], ids=["plain", "mix"])
def test_root_vectors(mix):
    case, expm = sweep_joint_case(48, False, mix)
    D = case.w.D
    rng = np.random.default_rng(48)
    sparse = np.zeros(D)
    keep = np.sort(rng.permutation(D)[:D // 3])
    sparse[keep] = rng.dirichlet(np.full(len(keep), 2.0))
    roots = {"dirichlet": case.root, "uniform": np.full(D, 1.0 / D), "sparse": sparse}
    lf = new_lf(case)
    got = {}
    for name, root in roots.items():
        got[name] = joint_call(lf, case, root=root)
        check_agreement(*got[name], case_args(case, expm, root=root), range(case.n), f"root {name} mix={mix}")
    assert np.all(np.isin(got["sparse"][0][:, -1], keep))
    st, jl = joint_call(lf, case, root=np.zeros(D))
    lf.close()
    assert np.all(st[:, -1] == 0) and np.all(jl == -np.inf)


# ---------------------------------------------------------------------------------------------------------------------
# 5. exact ties, 6. gaps
# ---------------------------------------------------------------------------------------------------------------------
def test_exact_ties():
    case, expm, cols = tie_joint_case()
    lf = new_lf(case)
    D = case.w.D
    pi = np.random.default_rng(5).dirichlet(np.full(D, 2.0))
    site = lf.part.batch_site_likelihoods(case.pats[:1], case.V[:1], pi)
    print(f"[ties] constant column: siteLnL - log pi_7 = {site[0] - np.log(pi[7]):.2e}")
    assert abs(site[0] - np.log(pi[7])) <= 1e-15
    st, jl = joint_call(lf, case)
    lf.close()
    assert np.all(st[0] == 7) and np.all(st[1] == 3) and st[2][-1] == 0 and jl[2] == -np.inf and np.all(st[3] == 5)
    for k in range(len(cols)):
        ref, l_star, _ = jr.joint_states(*case_args(case, expm, cols)(k))
        assert np.array_equal(st[k], ref) and (jl[k] == float(l_star) or abs(jl[k] - float(l_star)) <= 1e-15), k


def test_gaps():
    case, expm, cols = gap_joint_case()
    cherry, _ = leaf_cherry(case.w.tree)
    lf = new_lf(case)
    st, jl = joint_call(lf, case, V=case.V[:3], pats=np.arange(3))
    lf.close()
    assert np.all(st[0] == -1) and jl[0] == 0.0
    assert st[1][cherry] == -1 and (st[1] >= 0).sum() == case.w.tree.n_internal - 1
    assert np.all(st[2] >= 0)
    check_agreement(st, jl, case_args(case, expm, cols), range(3), "gaps")


# ---------------------------------------------------------------------------------------------------------------------
# 8. bad input, chunks
# ---------------------------------------------------------------------------------------------------------------------
def test_nan_stays_in_its_set():
    for mix in (False, True):
        case, _ = sweep_joint_case(61, True, mix)
        lf = new_lf(case)
        clean = joint_call(lf, case)
        V = case.V.copy()
        V[3, 1, 0] = np.nan
        W = None
        if mix:
            W = case.W.copy()
            W[7, 2] = np.nan
        st, jl = joint_call(lf, case, V=V, W=W)
        lf.close()
        bad = [3, 7] if mix else [3]
        assert np.all(np.isnan(jl[bad])) and np.all((st[bad] >= -1) & (st[bad] < case.w.D))
        others = ~np.isin(np.arange(case.n), bad)
        assert np.array_equal(st[others], clean[0][others]) and np.array_equal(jl[others], clean[1][others])


@pytest.mark.parametrize("mix", [False, True], ids=["plain", "mix"])
def test_chunks_match_small_calls(mix):
    w, _ = gc.load("mg94_8x60_c1")
    rng = np.random.default_rng(44 + mix)
    n = 1100
    branch_k, V, W, _ = meme_sets(w, 2, n, rng)
    if not mix:
        off = np.concatenate([[0], np.cumsum(branch_k)])
        V, W, branch_k = np.ascontiguousarray(V[:, off[:-1]]), None, None
    pats = rng.integers(0, w.S, n)
    lf = LF(w)

    def call(sl):
        return lf.part.batch_joint_ancestors(pats[sl], V[sl], w.pi, weights=None if W is None else W[sl],
                                             branch_k=branch_k, want_site=True)
    full = call(slice(0, n))
    a, b = call(slice(0, 1024)), call(slice(1024, n))
    for x, y, z in zip(full, a, b):
        assert np.array_equal(x, np.concatenate([y, z]))
    assert np.all(full[0] >= 0) and np.all(np.isfinite(full[1]))
    for s in (0, 1023, 1024, n - 1):
        one = call(slice(s, s + 1))
        assert np.array_equal(one[0][0], full[0][s]) and one[1][0] == full[1][s]
    again = call(slice(0, n))
    lf.close()
    assert all(np.array_equal(x, y) for x, y in zip(full, again))


# ---------------------------------------------------------------------------------------------------------------------
# 9. non-interference, refusals
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("flags", [engine.FLAG_FORCE_FP64, engine.FLAG_DEFAULT])
def test_no_interference(flags):
    w, _ = gc.load("mg94_30x100_c4_ambig")
    rng = np.random.default_rng(45)
    lf = LF(w, flags)
    part = lf.part
    lf.set_all_matrices()
    before = lf.compute()
    part.branch_cache_build(5, w.pi)
    bc0 = part.branch_cache_evaluate(w.class_weights)
    branch_k, V, W, _ = meme_sets(w, 3, 40, rng)
    pats = rng.choice(w.S, 40)
    off = np.concatenate([[0], np.cumsum(branch_k)])
    Vp = np.ascontiguousarray(V[:, off[:-1]])
    sup0 = part.batch_leaf_support(pats, V, w.pi, weights=W, branch_k=branch_k, want_site=True)
    rows0 = part.batch_branch_component_likelihoods(pats, V, W, w.pi, branch_k=branch_k)
    plain0 = part.batch_site_likelihoods(pats, Vp, w.pi)
    a = part.batch_joint_ancestors(pats, V, w.pi, weights=W, branch_k=branch_k, want_site=True)
    assert part.branch_cache_evaluate(w.class_weights) == bc0
    sup = part.batch_leaf_support(pats, V, w.pi, weights=W, branch_k=branch_k, want_site=True)
    b = part.batch_joint_ancestors(pats, Vp, w.pi, want_site=True)
    part.batch_site_simulate(Vp[:4], w.pi, 3)
    assert np.array_equal(part.batch_site_likelihoods(pats, Vp, w.pi), plain0)
    assert np.array_equal(part.batch_branch_component_likelihoods(pats, V, W, w.pi, branch_k=branch_k)[1], rows0[1])
    c = part.batch_joint_ancestors(pats, V, w.pi, weights=W, branch_k=branch_k, want_site=True)
    assert np.array_equal(part.batch_leaf_support(pats, V, w.pi, weights=W, branch_k=branch_k, want_site=True)[0], sup0[0])
    assert part.branch_cache_evaluate(w.class_weights) == bc0
    assert lf.compute() == before
    lf.close()
    assert np.array_equal(sup[0], sup0[0]) and np.array_equal(sup[1], sup0[1])
    assert all(np.array_equal(x, y) for x, y in zip(a, c))
    assert np.array_equal(b[2], plain0) and np.array_equal(a[2], sup0[1]) and np.all(b[0] >= 0)


def _raw(part, pats, K, branch_k, V, W, root, site, jl, st):
    po, ppo = _i(pats)
    pbk = None if branch_k is None else _i(branch_k)[1]
    pv = None if V is None else _d(V)[1]
    pw = None if W is None else _d(W)[1]
    ppi = None if root is None else _d(root)[1]
    ps = None if site is None else site.ctypes.data_as(_dp)
    pj = None if jl is None else jl.ctypes.data_as(_dp)
    pst = None if st is None else st.ctypes.data_as(_ip)
    return part._lib.hb2_batch_joint_ancestors(part._h, 0, len(po), ppo, int(K), pbk, pv, pw, None, ppi, ps, pj, pst)


def test_refusals_leave_partition_usable():
    w, _ = gc.load("mg94_8x60_c1")
    rng = np.random.default_rng(46)
    branch_k, V, W, _ = meme_sets(w, 2, 8, rng)
    off = np.concatenate([[0], np.cumsum(branch_k)])
    Vp = np.ascontiguousarray(V[:, off[:-1]])
    pats = rng.choice(w.S, 8, replace=False)
    I = w.tree.n_internal
    lf = LF(w)
    lf.set_all_matrices()
    lnl = lf.compute()
    good = lf.part.batch_joint_ancestors(pats, V, w.pi, weights=W, branch_k=branch_k)
    good_p = lf.part.batch_joint_ancestors(pats, Vp, w.pi)
    bad_k, bad_pat = branch_k.copy(), pats.copy()
    bad_k[0] = 3
    bad_pat[2] = w.S
    cases = [((pats, 0, branch_k, V, W, w.pi), "K=0 outside 1..4"), ((pats, 5, branch_k, V, W, w.pi), "K=5 outside 1..4"),
             ((pats, 2, bad_k, V, W, w.pi), r"branchK\[0\]=3 outside 1..2"),
             ((pats, 2, None, Vp, None, w.pi), "K=2 and branchK need weights"),
             ((pats, 1, branch_k, Vp, None, w.pi), "K=1 and branchK need weights"),
             ((pats, 2, branch_k, None, W, w.pi), "null argument"), ((pats, 2, branch_k, V, W, None), "null argument"),
             ((pats, 1, None, None, None, w.pi), "null argument"),
             ((bad_pat, 2, branch_k, V, W, w.pi), rf"patternOf\[2\]={w.S} out of range"),
             ((bad_pat, 1, None, Vp, None, w.pi), rf"patternOf\[2\]={w.S} out of range")]
    for args, msg in cases:
        site, jl, st = np.full(8, 7.0), np.full(8, 7.0), np.full((8, I), 7, np.int64)
        assert _raw(lf.part, *args, site, jl, st) != 0
        assert re.search(msg, lf.part._lib.hb2_last_error().decode()), lf.part._lib.hb2_last_error()
        assert np.all(site == 7.0) and np.all(jl == 7.0) and np.all(st == 7)
    for args in ((pats, 2, branch_k, V, W, w.pi), (pats, 1, None, Vp, None, w.pi)):
        site, jl = np.full(8, 7.0), np.full(8, 7.0)
        assert _raw(lf.part, *args, site, jl, None) != 0
        assert "nodeStates must not be null" in lf.part._lib.hb2_last_error().decode()
        assert np.all(site == 7.0) and np.all(jl == 7.0)
    # siteLnL and jointLnL are nullable
    st = np.empty((8, I), np.int64)
    _check(_raw(lf.part, pats, 2, branch_k, V, W, w.pi, None, None, st))
    assert np.array_equal(st, good[0])
    _check(_raw(lf.part, pats, 1, None, Vp, None, w.pi, None, None, st))
    assert np.array_equal(st, good_p[0])
    # nSets == 0 does nothing
    _check(_raw(lf.part, pats[:0], 2, branch_k, V[:0], W[:0], w.pi, np.empty(0), np.empty(0), np.empty((0, I), np.int64)))
    again = lf.part.batch_joint_ancestors(pats, V, w.pi, weights=W, branch_k=branch_k)
    assert all(np.array_equal(x, y) for x, y in zip(again, good))
    assert lf.compute() == lnl
    lf.close()
    # 20 states: refused like the other batch entry points, and the partition still evaluates
    w20 = tree_workload(flat_tree(star(5)), 20, 40)
    lf = LikelihoodFunction(w20, flags=engine.FLAG_FORCE_FP64)
    lf.set_all_matrices()
    lnl = lf.compute()
    nb = w20.tree.n_branches
    st = np.full((1, 1), 7, np.int64)
    assert _raw(lf.part, [0], 1, None, np.zeros((1, nb, 4)), None, w20.pi, np.empty(1), np.empty(1), st) != 0
    assert "33..64-state" in lf.part._lib.hb2_last_error().decode()
    assert np.all(st == 7)
    assert lf.compute() == lnl
    lf.close()
