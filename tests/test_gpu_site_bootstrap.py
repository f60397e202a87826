"""GPU suite (pytest -m gpu): the site-level parametric bootstrap of FEL and MEME (--resample).  hb2_batch_site_simulate
draws replicate columns from each set's own model; hb2_batch_column_likelihoods scores caller-given columns.  Checked
draw by draw against the oracle's matrices, for invariance under chunking and splitting, against the pattern entry
points, against the oracle's likelihoods of the simulated columns, for isolation from the resident state, and for every
refusal."""
import dataclasses
import re

import numpy as np
import pytest

from hyphy_b200 import LikelihoodFunction, engine
from hyphy_b200.engine import EngineError, _check, _d, _i, _dp, _ip
from oracle import port
from tests import golden_cases as gc
from tests import simulate_reference as sim_ref
from tests import site_bootstrap_reference as ref
from tests.test_gpu_batch_mixture import meme_sets, dense, oracle_set
from tests.test_gpu_shapes import flat_tree, star, tree_workload

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _need_gpu(engine_lib):
    assert engine.device_count() > 0, "GPU tests need a CUDA device (no fallback exists)"


def LF(w, flags=engine.FLAG_FORCE_FP64):
    lf = LikelihoodFunction(w, flags=flags)
    lf.set_template()
    return lf


def fel_sets(w, n, rng):
    """FEL-shaped sets: one row per branch, tested / background branches as the group hint.  (formula values [n, B, nF],
    branch groups [B])"""
    _, V, _, tested = meme_sets(w, 1, n, rng)
    return V, tested.astype(np.int64)


def oracle_P(w, branch_k, v, wt):
    """Per-branch transition matrices [B, D, D] of one set: port.expm of every row, mixed in component order."""
    P = np.stack([port.expm(dense(w, v[r]), True) for r in range(len(v))])
    return ref.mix(P, wt, branch_k)


ROOT_SEED = 11


def root_freqs(w):
    return np.random.default_rng(ROOT_SEED).dirichlet(np.full(w.D, 4.0))


# ---------------------------------------------------------------------------------------------------------------------
# 1. draw by draw against the oracle's matrices
# ---------------------------------------------------------------------------------------------------------------------
def test_draws_match_oracle_rows():
    """Every child state, given the engine's own parent state, is the reference draw from the oracle's matrix row on the
    stated uniform.  The engine's matrices agree with the oracle's to ~1e-13, so a draw whose u*T lies within 1e-11*T of
    a prefix boundary may go either way: those are counted, and there must be few."""
    w, _ = gc.load("c2_mg94_50x1000_c1")
    rng = np.random.default_rng(21)
    n_sets, n_reps, seed, first_set, first_rep = 8, 500, 0xC0FFEE1234, 40, 3000
    pi = root_freqs(w)
    fel_V, fel_bg = fel_sets(w, n_sets, rng)
    bk, V, W, tested = meme_sets(w, 2, n_sets, rng)
    lf = LF(w)
    L, I, B = w.tree.n_leaves, w.tree.n_internal, w.tree.n_branches
    fp = w.tree.flat_parents
    near = 0
    for shape, (vals, wts, branch_k, bg) in {"fel": (fel_V, None, None, fel_bg), "meme": (V, W, bk, tested.astype(np.int64))}.items():
        leaf, nodes = lf.part.batch_site_simulate(vals, pi, n_reps, weights=wts, branch_k=branch_k, branch_group=bg, seed=seed,
                                                  first_set=first_set, first_rep=first_rep, want_nodes=True)
        assert leaf.shape == (n_sets, n_reps, L) and nodes.shape == (n_sets, n_reps, I)
        g = np.arange(first_rep, first_rep + n_reps, dtype=np.uint64)
        rc, rl = sim_ref.prefix(pi)
        for s in range(n_sets):
            t = np.uint64(first_set + s)
            state = np.concatenate([leaf[s], nodes[s]], axis=1).T          # [L+I, n_reps], flat order
            u = ref.uniforms(g, L + I - 1, t, seed)
            assert np.array_equal(state[-1], sim_ref.draw(np.broadcast_to(rc, (n_reps, w.D)), np.full(n_reps, rl), u))
            P = oracle_P(w, np.ones(B, np.int64) if branch_k is None else branch_k, vals[s], np.ones(vals.shape[1]) if wts is None else wts[s])
            cdf, last = sim_ref.prefix(P)
            for node in range(L + I - 1):
                par = state[L + fp[node]]
                u = ref.uniforms(g, node, t, seed)
                c = cdf[node, par]
                want = sim_ref.draw(c, last[node, par], u)
                bad = np.nonzero(state[node] != want)[0]
                if len(bad):
                    T = c[bad, -1]
                    gap = np.abs(c[bad] - (u[bad] * T)[:, None]).min(axis=1)
                    assert np.all(gap <= 1e-11 * T), (shape, s, node, bad, state[node][bad], want[bad])
                    near += len(bad)
    lf.close()
    print(f"draws within 1e-11*T of a prefix boundary that differ from the oracle's: {near}")
    assert near <= 5


# ---------------------------------------------------------------------------------------------------------------------
# 2. chunking and splitting are invisible
# ---------------------------------------------------------------------------------------------------------------------
def test_chunks_and_splits_are_invisible():
    w, _ = gc.load("mg94_8x60_c1")
    rng = np.random.default_rng(22)
    n, reps, seed = 1100, 7, 99                                          # > 1024 sets: the engine chunks
    pi = root_freqs(w)
    bk, V, W, tested = meme_sets(w, 2, n, rng)
    fel_V, fel_bg = fel_sets(w, n, rng)
    lf = LF(w)
    for kw in (dict(formula_values=V, weights=W, branch_k=bk), dict(formula_values=fel_V, branch_group=fel_bg)):
        vals = kw.pop("formula_values")
        wts = kw.pop("weights", None)

        def sim(lo, hi, r0, nr):
            return lf.part.batch_site_simulate(vals[lo:hi], pi, nr, weights=None if wts is None else wts[lo:hi], seed=seed,
                                               first_set=lo, first_rep=r0, want_nodes=True, **kw)

        whole = sim(0, n, 0, reps)
        by_sets = [sim(lo, min(lo + 300, n), 0, reps) for lo in range(0, n, 300)]
        by_reps = [sim(0, n, 0, 3), sim(0, n, 3, reps - 3)]
        for k in range(2):
            assert np.array_equal(whole[k], np.concatenate([p[k] for p in by_sets], axis=0))
            assert np.array_equal(whole[k], np.concatenate([p[k] for p in by_reps], axis=1))
        assert len(np.unique(whole[0].reshape(n * reps, -1), axis=0)) > n          # columns differ across sets and replicates
        # the same call again, and a call without internal states, give the same leaves
        assert np.array_equal(sim(0, n, 0, reps)[0], whole[0])
        assert np.array_equal(lf.part.batch_site_simulate(vals, pi, reps, weights=wts, seed=seed, **kw)[0], whole[0])
    lf.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3. the partition's own patterns as columns
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["mg94_8x60_c4_ambig", "mg94_30x100_c4_ambig"])
def test_columns_equal_patterns(name):
    w, _ = gc.load(name)
    rng = np.random.default_rng(23)
    n = 1300                                                             # two chunks
    pats = rng.integers(0, w.S, n)
    cols = np.ascontiguousarray(w.leaf_states[:, pats].T)
    assert (cols < 0).any()
    pi = root_freqs(w)
    lf = LF(w)
    fel_V, fel_bg = fel_sets(w, n, rng)
    for bg in (fel_bg, None):
        want = lf.part.batch_site_likelihoods(pats, fel_V, pi, branch_group=bg)
        assert np.array_equal(lf.part.batch_column_likelihoods(cols, fel_V, pi, branch_group=bg), want)
    bk, V, W, tested = meme_sets(w, 3, n, rng)
    for bg in (tested.astype(np.int64), None):
        want = lf.part.batch_site_mixture_likelihoods(pats, V, W, pi, branch_k=bk, branch_group=bg)
        assert np.all(np.isfinite(want))
        assert np.array_equal(lf.part.batch_column_likelihoods(cols, V, pi, weights=W, branch_k=bk, branch_group=bg), want)
    lf.close()


# ---------------------------------------------------------------------------------------------------------------------
# 4. simulated columns scored against the oracle
# ---------------------------------------------------------------------------------------------------------------------
def test_simulated_columns_match_oracle():
    w, _ = gc.load("c2_mg94_50x1000_c1")
    rng = np.random.default_rng(24)
    n, reps = 5, 2
    pi = w.pi                                                            # the oracle's root vector is the workload's
    B = w.tree.n_branches
    fel_V, fel_bg = fel_sets(w, n, rng)
    bk, V, W, tested = meme_sets(w, 2, n, rng)
    lf = LF(w)
    for vals, wts, branch_k, bg in ((fel_V, None, None, fel_bg), (V, W, bk, tested.astype(np.int64))):
        leaf, _ = lf.part.batch_site_simulate(vals, pi, reps, weights=wts, branch_k=branch_k, branch_group=bg, seed=7)
        cols = leaf.reshape(n * reps, -1)
        rv = np.repeat(vals, reps, axis=0)
        rw = None if wts is None else np.repeat(wts, reps, axis=0)
        got = lf.part.batch_column_likelihoods(cols, rv, pi, weights=rw, branch_k=branch_k, branch_group=bg)
        wc = dataclasses.replace(w, leaf_states=cols.T.copy(), ambig=np.zeros((0, w.D)), pattern_freq=np.ones(n * reps, dtype=np.int64),
                                 site_to_pattern=np.arange(n * reps), site_chars=None)
        k = np.ones(B, np.int64) if branch_k is None else branch_k
        want = np.array([oracle_set(wc, i, k, rv[i], np.ones(rv.shape[1]) if rw is None else rw[i]) for i in range(n * reps)])
        assert np.all(np.isfinite(want))
        assert np.all(np.abs(got - want) <= 1e-10 * np.abs(want)), (got, want)
    lf.close()


# ---------------------------------------------------------------------------------------------------------------------
# 5. no interference with the resident state
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("flags", [engine.FLAG_FORCE_FP64, engine.FLAG_DEFAULT])
def test_resident_state_untouched(flags):
    """evaluate -> simulate / score -> evaluate is bit-identical, and a branch cache built before the calls still serves
    after them, although the batch calls use another root vector."""
    w, _ = gc.load("mg94_8x60_c4_ambig")
    rng = np.random.default_rng(25)
    lf = LF(w, flags)
    lf.set_all_matrices()
    before = lf.compute(want_sites=True)
    lf.part.branch_cache_build(3, w.pi)
    cached = lf.part.branch_cache_evaluate(weights=w.class_weights, want_sites=True)
    pi = root_freqs(w)
    assert not np.allclose(pi, w.pi)
    bk, V, W, _ = meme_sets(w, 2, 20, rng)
    leaf, _ = lf.part.batch_site_simulate(V, pi, 6, weights=W, branch_k=bk, seed=3, want_nodes=True)
    lf.part.batch_column_likelihoods(leaf.reshape(120, -1), np.repeat(V, 6, axis=0), pi, weights=np.repeat(W, 6, axis=0), branch_k=bk)
    after = lf.part.branch_cache_evaluate(weights=w.class_weights, want_sites=True)
    for x, y in zip(cached, after):
        assert np.array_equal(x, y)
    again = lf.compute(want_sites=True)
    for x, y in zip(before, again):
        assert np.array_equal(x, y)
    lf.close()


# ---------------------------------------------------------------------------------------------------------------------
# 6. refusals
# ---------------------------------------------------------------------------------------------------------------------
def _raw_sim(part, n_sets, K, branch_k, V, W, bg, root, n_reps, first_set, first_rep, leaf, template=0):
    """The C entry point with arguments the Python wrapper would not let through."""
    p = lambda a, f: None if a is None else f(a)[1]                     # noqa: E731
    return part._lib.hb2_batch_site_simulate(part._h, template, n_sets, K, p(branch_k, _i), p(V, _d), p(W, _d), p(bg, _i),
                                             p(root, _d), n_reps, 5, first_set, first_rep,
                                             None if leaf is None else leaf.ctypes.data_as(_ip), None)


def _raw_cols(part, cols, K, branch_k, V, W, root, out):
    p = lambda a, f: None if a is None else f(a)[1]                     # noqa: E731
    return part._lib.hb2_batch_column_likelihoods(part._h, 0, len(V), p(cols, _i), K, p(branch_k, _i), p(V, _d), p(W, _d), None,
                                                  p(root, _d), out.ctypes.data_as(_dp))


def _refused(rc, lib, msg):
    assert rc != 0
    err = lib.hb2_last_error().decode()
    assert re.search(msg, err), err


def test_refusals():
    w, _ = gc.load("mg94_8x60_c1")
    rng = np.random.default_rng(26)
    lf = LF(w)
    lf.set_all_matrices()
    lnl = lf.compute()
    lib = lf.part._lib
    n, reps = 4, 3
    pi = root_freqs(w)
    bk, V, W, _ = meme_sets(w, 2, n, rng)
    fel_V, _ = fel_sets(w, n, rng)
    good, _ = lf.part.batch_site_simulate(V, pi, reps, weights=W, branch_k=bk, seed=5)
    B = w.tree.n_branches
    big_k = bk.copy()
    big_k[0] = 3
    bad_bg = np.zeros(B, np.int64)
    bad_bg[2] = 8
    zero_pi, neg_pi, nan_pi = np.zeros(w.D), pi.copy(), pi.copy()
    neg_pi[4], nan_pi[7] = -0.1, np.nan
    cases = [  # (n_sets, K, branch_k, V, W, bg, root, n_reps, first_set, first_rep), message
        ((n, 2, bk, V, W, None, pi, reps, 0, 0, 7), "template 7 has not been defined"),
        ((n, 2, bk, V, None, None, pi, reps, 0, 0), "K=2 and branchK need weights"),
        ((n, 1, bk, fel_V, None, None, pi, reps, 0, 0), "K=1 and branchK need weights"),
        ((n, 5, bk, V, W, None, pi, reps, 0, 0), "K=5 outside 1..4"),
        ((n, 2, big_k, V, W, None, pi, reps, 0, 0), r"branchK\[0\]=3 outside 1..2"),
        ((n, 2, bk, V, W, bad_bg, pi, reps, 0, 0), r"branchGroup\[2\]=8 outside 0..7"),
        ((n, 2, bk, None, W, None, pi, reps, 0, 0), "formulaValues must not be null"),
        ((n, 2, bk, V, W, None, None, reps, 0, 0), "rootFreqs must not be null"),
        ((-1, 2, bk, V, W, None, pi, reps, 0, 0), "nSets=-1 is negative"),
        ((n, 2, bk, V, W, None, pi, -2, 0, 0), "nReps=-2 is negative"),
        ((n, 2, bk, V, W, None, pi, reps, 0, -1), "firstRep=-1 out of range"),
        ((n, 2, bk, V, W, None, pi, reps, 0, 2 ** 63 - 2), "firstRep=9223372036854775806 out of range"),
        ((n, 2, bk, V, W, None, pi, reps, -1, 0), "firstSet=-1 out of range"),
        ((n, 2, bk, V, W, None, pi, reps, 2 ** 32 - 3, 0), "firstSet=4294967293 out of range"),
        ((n, 2, bk, V, W, None, zero_pi, reps, 0, 0), "root frequencies must be"),
        ((n, 2, bk, V, W, None, neg_pi, reps, 0, 0), "root frequencies must be"),
        ((n, 2, bk, V, W, None, nan_pi, reps, 0, 0), "root frequencies must be"),
    ]
    for args, msg in cases:
        leaf = np.full((n, reps, w.tree.n_leaves), -7, dtype=np.int64)
        _refused(_raw_sim(lf.part, *args[:10], leaf, *args[10:]), lib, msg)
        assert np.all(leaf == -7)                                        # a refused call writes nothing
    _refused(_raw_sim(lf.part, n, 2, bk, V, W, None, pi, reps, 0, 0, None), lib, "leafStates must not be null")
    # the largest admissible firstSet and firstRep are accepted
    leaf = np.empty((n, reps, w.tree.n_leaves), dtype=np.int64)
    _check(_raw_sim(lf.part, n, 2, bk, V, W, None, pi, reps, 2 ** 32 - n, 2 ** 63 - 1 - reps, leaf))
    # a set whose matrix has a bad row (NaN formula values) is named with its branch and row
    Vn = V.copy()
    Vn[2, 0] = np.nan
    with pytest.raises(EngineError, match="row 0 of the transition matrix of set 2, branch 0 does not"):
        lf.part.batch_site_simulate(Vn, pi, reps, weights=W, branch_k=bk)
    # column codes out of range, named with set and leaf; nothing written
    cols = good.reshape(n * reps, -1).copy()
    rv, rw = np.repeat(V, reps, axis=0), np.repeat(W, reps, axis=0)
    for code in (w.D, -(len(w.ambig) + 1)):
        bad = cols.copy()
        bad[5, 3] = code
        out = np.full(n * reps, -7.0)
        _refused(_raw_cols(lf.part, bad, 2, bk, rv, rw, pi, out), lib, f"set 5, leaf 3: code {code} is neither")
        assert np.all(out == -7.0)
    out = np.full(n * reps, -7.0)
    _refused(_raw_cols(lf.part, None, 2, bk, rv, rw, pi, out), lib, "columns must not be null")
    _refused(_raw_cols(lf.part, cols, 2, bk, rv, None, pi, out), lib, "K=2 and branchK need weights")
    assert np.all(out == -7.0)
    # the partition is still usable
    assert np.array_equal(lf.part.batch_site_simulate(V, pi, reps, weights=W, branch_k=bk, seed=5)[0], good)
    assert lf.compute() == lnl
    lf.close()
    # 20 states: refused like the other batch entry points
    w20 = tree_workload(flat_tree(star(5)), 20, 40)
    lf = LikelihoodFunction(w20, flags=engine.FLAG_FORCE_FP64)
    nb = w20.tree.n_branches
    leaf = np.full((1, 2, 5), -7, dtype=np.int64)
    _refused(_raw_sim(lf.part, 1, 1, None, np.zeros((1, nb, 4)), None, None, w20.pi, 2, 0, 0, leaf), lf.part._lib, "33..64-state")
    assert np.all(leaf == -7)
    lf.close()
