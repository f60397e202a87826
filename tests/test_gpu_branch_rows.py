"""GPU suite (pytest -m gpu): hb2_batch_branch_component_likelihoods, the likelihood of each set with each branch pinned
to each of its mixture components (MEME's branch-level empirical Bayes, MEME.bf:886-944), against the unmodified reference
binary's pinned per-site values, the long-double reference (tests/branch_rows_reference.py), the oracle, and the mixture
entry point fed one-hot weights -- MEME's own brute force, on the device."""
import re

import numpy as np
import pytest

from hyphy_b200 import LikelihoodFunction, engine
from hyphy_b200.engine import _check, _d, _i, _dp
from oracle import port
from tests import batch_reference as br
from tests import branch_rows_reference as brr
from tests import golden_cases as gc
from tests.test_gpu_batch_mixture import LF, dense, meme_sets, one_pattern, oracle_set, with_omegas
from tests.test_gpu_shapes import TREES, flat_tree, longdouble_sites, star, tree_workload, underflow_workload

pytestmark = pytest.mark.gpu

TOL = 1e-10                 # relative, as test_gpu_batch_mixture.py (plus 1e-12 absolute)
TOL_BRUTE = 1e-11           # against the mixture entry point with one-hot weights


@pytest.fixture(scope="module", autouse=True)
def _need_gpu(engine_lib):
    assert engine.device_count() > 0, "GPU tests need a CUDA device (no fallback exists)"


class CodonExpm:
    """Exponential of one row of a codon workload's compiled formula values, once per distinct row: expm_ld (long double)
    or the oracle's port.expm (fp64)."""

    def __init__(self, w, ld):
        self.w, self.ld, self.memo = w, ld, {}

    def __call__(self, v):
        key = np.asarray(v, dtype=np.float64).tobytes()
        if key not in self.memo:
            M = dense(self.w, v)
            self.memo[key] = br.expm_ld(M.astype(br.LD)) if self.ld else np.asarray(port.expm(M, True), dtype=br.LD)
        return self.memo[key]


def offsets(branch_k):
    return np.concatenate([[0], np.cumsum(branch_k)]).astype(np.int64)


def one_hot(branch_k, W):
    """Per (set, row): the set's weights with the row's branch one-hot on the row's component -> [n * R, R]."""
    off = offsets(branch_k)
    n, R = W.shape
    out = np.repeat(W, R, axis=0).reshape(n, R, R)
    for b in range(len(branch_k)):
        for r in range(off[b], off[b + 1]):
            out[:, r, off[b]:off[b + 1]] = 0.0
            out[:, r, r] = 1.0
    return out.reshape(n * R, R)


def brute_force(part, w, pats, branch_k, V, W):
    """rows [n, R] by the mixture entry point, one set per (set, row) with one-hot weights on the row's branch."""
    n, R = W.shape
    got = part.batch_site_mixture_likelihoods(np.repeat(pats, R), np.repeat(V, R, axis=0), one_hot(branch_k, W), w.pi,
                                              branch_k=branch_k)
    return got.reshape(n, R)


def mixture_identity(branch_k, W, site, rows):
    """log sum_k w_k exp(l_{b,k} - l_s) for every (set, branch) -> [n, B]."""
    off = offsets(branch_k)
    return np.stack([np.log((W[:, off[b]:off[b + 1]] * np.exp(rows[:, off[b]:off[b + 1]] - site[:, None])).sum(axis=1))
                     for b in range(len(branch_k))], axis=1)


def oracle_rows(w, pattern, branch_k, v, wt, r):
    """oracle_set (port.expm per row, the weighted sum in component order, port.prune) with row r's branch one-hot."""
    off = offsets(branch_k)
    b = int(np.searchsorted(off, r, side="right") - 1)
    hot = wt.copy()
    hot[off[b]:off[b + 1]] = 0.0
    hot[r] = 1.0
    return oracle_set(w, pattern, branch_k, v, hot)


def all_tested(w, K, n, rng):
    """MEME-shaped sets as meme_sets draws them, with every branch tested: (branch_k [B], V [n, R, nF], W [n, R])."""
    nb = w.tree.n_branches
    unit = with_omegas(w, [1.0]).compiled_values()[0]
    nonsyn = ~np.isclose(with_omegas(w, [2.0]).compiled_values()[0][0], unit[0])
    V = np.empty((n, nb * K, unit.shape[1]))
    W = np.empty((n, nb * K))
    for i in range(n):
        alpha = rng.uniform(0.2, 3.0)
        betas = np.sort(rng.uniform(0.0, 10.0, K))
        wk = rng.dirichlet(np.ones(K))
        for b in range(nb):
            for k in range(K):
                V[i, b * K + k] = unit[b] * np.where(nonsyn, betas[k], alpha)
                W[i, b * K + k] = wk[k]
    return np.full(nb, K, dtype=np.int64), V, W


# ---------------------------------------------------------------------------------------------------------------------
# 1. the reference binary's pinned values
# ---------------------------------------------------------------------------------------------------------------------
def test_pinned_fixture_matches_reference():
    """Every site of bsrel_12x80_k3, K = 3 on every branch, each branch pinned to each component by one-hot local weights
    in the unmodified reference binary (tools/make_golden.py --pinned)."""
    w, _ = gc.load("bsrel_12x80_k3")
    g = np.load(gc.GOLDEN_DIR + "/bsrel_12x80_k3_pinned.npz")
    assert str(g["checksum"]) == gc.checksum(w)
    mix = w.meta["mixture"]
    K, nb = len(mix["omegas"]), w.tree.n_branches
    comp = with_omegas(w, mix["omegas"]).compiled_values()
    rows = comp.transpose(1, 0, 2).reshape(nb * K, -1)
    pats = np.arange(w.S)
    lf = LF(w)
    site, got = lf.part.batch_branch_component_likelihoods(pats, np.broadcast_to(rows, (w.S,) + rows.shape),
                                                           np.tile(mix["weights"], (w.S, nb)), w.pi)
    lf.close()
    assert np.abs(site[w.site_to_pattern] - g["site_lnL"]).max() <= 1e-9
    err = np.abs(got[w.site_to_pattern].T - g["pinned"])
    assert err.max() <= 1e-9, err.max()


# ---------------------------------------------------------------------------------------------------------------------
# 2. MEME-shaped sets: long-double reference, oracle, brute force on the device; 3. identities
# ---------------------------------------------------------------------------------------------------------------------
MEME_CASES = [(name, K, layout) for name in ("c2_mg94_50x1000_c1", "mg94_30x100_c4_ambig") for K in (2, 3, 4)
              for layout in ("third", "all")]


@pytest.mark.parametrize("name,K,layout", MEME_CASES)
def test_meme_sets(name, K, layout):
    w, _ = gc.load(name)
    rng = np.random.default_rng(10 * K + len(name) + (layout == "all"))
    n = 3
    if layout == "third":
        branch_k, V, W, _ = meme_sets(w, K, n, rng)
    else:
        branch_k, V, W = all_tested(w, K, n, rng)
    if len(w.ambig):
        amb = np.nonzero((w.leaf_states < 0).any(axis=0))[0]
        pats = np.concatenate([amb[:1], rng.choice(w.S, n - 1, replace=False)])
        assert (w.leaf_states[:, pats] < 0).any()
    else:
        pats = rng.choice(w.S, n, replace=False)
    lf = LF(w)
    site, rows = lf.part.batch_branch_component_likelihoods(pats, V, W, w.pi, branch_k=branch_k)
    mixed = lf.part.batch_site_mixture_likelihoods(pats, V, W, w.pi, branch_k=branch_k)
    brute = brute_force(lf.part, w, pats, branch_k, V, W)
    lf.close()
    assert np.all(np.isfinite(rows))
    assert np.array_equal(site, mixed)                                      # the same inside pass, bit for bit
    assert np.all(np.abs(rows - brute) <= TOL_BRUTE * np.abs(brute)), np.abs(rows - brute).max()
    assert np.abs(mixture_identity(branch_k, W, site, rows)).max() <= 1e-11
    one = branch_k == 1
    if one.any():
        r1 = offsets(branch_k)[:-1][one]
        assert np.all(np.abs(rows[:, r1] - site[:, None]) <= 1e-12 * np.abs(site[:, None]))
    # the long-double reference on the first set (the one with an ambiguous leaf), every row
    col = w.leaf_states[:, pats[0]]
    ref = brr.brute_rows(w.tree, CodonExpm(w, True), V[0], W[0], branch_k, col, w.ambig, w.pi).astype(np.float64)
    assert np.all(np.abs(rows[0] - ref) <= TOL * np.abs(ref) + 1e-12), np.abs(rows[0] - ref).max()
    # the oracle (port.expm + port.prune, one-hot weights on the row's branch) on 4 seeded rows of every set
    for i in range(n):
        for r in rng.choice(W.shape[1], 4, replace=False):
            want = oracle_rows(w, pats[i], branch_k, V[i], W[i], r)
            assert abs(rows[i, r] - want) <= TOL * abs(want) + 1e-12, (i, r, rows[i, r], want)


# ---------------------------------------------------------------------------------------------------------------------
# 4. tree shapes: deep and wide trees, a leaf under the root
# ---------------------------------------------------------------------------------------------------------------------
def _pinned_ld(w, pat, branch_k, V, W, rows_to_check):
    """Long-double pruning (longdouble_sites) of the oracle's exponentials with the row's branch pinned."""
    ex = CodonExpm(w, False)
    off = offsets(branch_k)
    nb = w.tree.n_branches
    E = [np.asarray(ex(V[r]), dtype=np.float64) for r in range(off[-1])]
    P = np.stack([sum(W[r] * E[r] for r in range(off[b], off[b + 1])) for b in range(nb)])
    w1 = one_pattern(w, pat)
    out = {}
    for r in rows_to_check:
        b = int(np.searchsorted(off, r, side="right") - 1)
        Pr = P.copy()
        Pr[b] = E[r]
        out[r] = float(longdouble_sites(w1, Pr)[0])
    return out


@pytest.mark.parametrize("shape", ["codon400", "caterpillar700", "star40", "poly7", "all_internal", "leaf_by_deep"])
def test_tree_shapes(shape):
    if shape == "codon400":
        w = underflow_workload("codon400")            # the 400-leaf star whose product falls below 2^-1022
    else:
        w = tree_workload(flat_tree(TREES[shape], mean_t=0.2, seed=len(shape)), 61, 150, seed=9)
    root_kids = w.tree.children()[-1]
    assert any(c < w.tree.n_leaves for c in root_kids)                         # a leaf directly under the root
    rng = np.random.default_rng(len(shape))
    n = 2
    branch_k, V, W, tested = meme_sets(w, 2, n, rng)
    pats = rng.choice(w.S, n, replace=False)
    lf = LF(w)
    site, rows = lf.part.batch_branch_component_likelihoods(pats, V, W, w.pi, branch_k=branch_k)
    assert np.array_equal(site, lf.part.batch_site_mixture_likelihoods(pats, V, W, w.pi, branch_k=branch_k))
    lf.close()
    assert np.all(np.isfinite(rows))
    assert np.abs(mixture_identity(branch_k, W, site, rows)).max() <= 1e-11
    off = offsets(branch_k)
    tested_rows = [r for b in np.nonzero(tested)[0] for r in range(off[b], off[b + 1])]
    check = sorted(set(tested_rows[:24]) | set(rng.choice(off[-1], 8, replace=False).tolist()))
    for i in range(n):
        ref = _pinned_ld(w, pats[i], branch_k, V[i], W[i], check)
        for r, want in ref.items():
            assert abs(rows[i, r] - want) <= TOL * abs(want) + 1e-12, (i, r, rows[i, r], want)


# ---------------------------------------------------------------------------------------------------------------------
# 5. degenerate inputs
# ---------------------------------------------------------------------------------------------------------------------
def test_zero_weight_component_gets_its_pinned_value():
    w, _ = gc.load("mg94_30x100_c4_ambig")
    rng = np.random.default_rng(21)
    branch_k, V, W, tested = meme_sets(w, 3, 6, rng)
    off = offsets(branch_k)
    tb = np.nonzero(tested)[0]
    W[:, off[tb] + 1] = 0.0                                                  # component 1 of every tested branch
    pats = rng.choice(w.S, 6, replace=False)
    lf = LF(w)
    site, rows = lf.part.batch_branch_component_likelihoods(pats, V, W, w.pi, branch_k=branch_k)
    brute = brute_force(lf.part, w, pats, branch_k, V, W)
    lf.close()
    zero = off[tb] + 1
    assert np.all(np.isfinite(rows[:, zero]))
    assert np.all(np.abs(rows - brute) <= TOL_BRUTE * np.abs(brute))


def test_nan_weight_stays_in_its_set():
    w, _ = gc.load("mg94_8x60_c4_ambig")
    rng = np.random.default_rng(22)
    branch_k, V, W, tested = meme_sets(w, 2, 16, rng)
    pats = rng.choice(w.S, 16, replace=False)
    lf = LF(w)
    clean = lf.part.batch_branch_component_likelihoods(pats, V, W, w.pi, branch_k=branch_k)
    Wn = W.copy()
    Wn[5, offsets(branch_k)[np.nonzero(tested)[0][0]]] = np.nan
    site, rows = lf.part.batch_branch_component_likelihoods(pats, V, Wn, w.pi, branch_k=branch_k)
    lf.close()
    assert np.isnan(site[5]) and np.isnan(rows[5]).any()
    others = np.arange(16) != 5
    assert np.array_equal(site[others], clean[0][others]) and np.array_equal(rows[others], clean[1][others])


def test_zero_formula_values_give_identity():
    w, _ = gc.load("mg94_8x60_c1")
    rng = np.random.default_rng(23)
    branch_k, V, W, _ = meme_sets(w, 2, w.S, rng)
    lf = LF(w)
    site, rows = lf.part.batch_branch_component_likelihoods(np.arange(w.S), np.zeros_like(V), W, w.pi, branch_k=branch_k)
    lf.close()
    const = np.all(w.leaf_states == w.leaf_states[:1], axis=0) & (w.leaf_states[0] >= 0)
    assert const.any() and (~const).any()
    assert np.all(rows[~const] == -np.inf) and np.all(site[~const] == -np.inf)
    want = np.log(w.pi[w.leaf_states[0, const]])
    np.testing.assert_allclose(rows[const], np.broadcast_to(want[:, None], rows[const].shape), rtol=1e-12)


# ---------------------------------------------------------------------------------------------------------------------
# 6. chunking
# ---------------------------------------------------------------------------------------------------------------------
def test_chunks_match_small_calls():
    """More than 1024 sets (the chunk cap) in one call = the same sets in separate calls, bit for bit; the call runs
    exactly the launches of its two chunks as separate calls."""
    w, _ = gc.load("mg94_8x60_c1")
    rng = np.random.default_rng(24)
    n = 1100
    branch_k, V, W, _ = meme_sets(w, 2, n, rng)
    pats = rng.integers(0, w.S, n)
    lf = LF(w)
    part = lf.part
    l0 = part.launch_count
    site, rows = part.batch_branch_component_likelihoods(pats, V, W, w.pi, branch_k=branch_k)
    l1 = part.launch_count
    a = part.batch_branch_component_likelihoods(pats[:1024], V[:1024], W[:1024], w.pi, branch_k=branch_k)
    l2 = part.launch_count
    b = part.batch_branch_component_likelihoods(pats[1024:], V[1024:], W[1024:], w.pi, branch_k=branch_k)
    l3 = part.launch_count
    parts = [part.batch_branch_component_likelihoods(pats[s:s + 100], V[s:s + 100], W[s:s + 100], w.pi, branch_k=branch_k)
             for s in range(0, n, 100)]
    lf.close()
    assert l1 - l0 == (l2 - l1) + (l3 - l2)                                 # two chunks
    assert np.all(np.isfinite(rows))
    assert np.array_equal(site, np.concatenate([a[0], b[0]])) and np.array_equal(rows, np.concatenate([a[1], b[1]]))
    assert np.array_equal(site, np.concatenate([p[0] for p in parts]))
    assert np.array_equal(rows, np.concatenate([p[1] for p in parts]))


# ---------------------------------------------------------------------------------------------------------------------
# 7. non-interference
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("flags", [engine.FLAG_FORCE_FP64, engine.FLAG_DEFAULT])
def test_no_interference(flags):
    w, _ = gc.load("mg94_30x100_c4_ambig")
    rng = np.random.default_rng(25)
    lf = LF(w, flags)
    part = lf.part
    lf.set_all_matrices()
    before = lf.compute()
    part.branch_cache_build(5, w.pi)
    bc0 = part.branch_cache_evaluate(w.class_weights)
    branch_k, V, W, _ = meme_sets(w, 3, 40, rng)
    pats = rng.choice(w.S, 40)
    a = part.batch_branch_component_likelihoods(pats, V, W, w.pi, branch_k=branch_k)
    assert part.branch_cache_evaluate(w.class_weights) == bc0
    assert lf.compute() == before
    b = part.batch_branch_component_likelihoods(pats, V, W, w.pi, branch_k=branch_k)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    lf.close()


# ---------------------------------------------------------------------------------------------------------------------
# 8. refusals (class-group mode needs two ranks: tests/test_multigpu.py's territory, not exercised here)
# ---------------------------------------------------------------------------------------------------------------------
def _raw(part, pats, K, branch_k, V, W, root, site, rows):
    po, ppo = _i(pats)
    pbk = None if branch_k is None else _i(branch_k)[1]
    pv = None if V is None else _d(V)[1]
    pw = None if W is None else _d(W)[1]
    ppi = None if root is None else _d(root)[1]
    ps = None if site is None else site.ctypes.data_as(_dp)
    pr = None if rows is None else rows.ctypes.data_as(_dp)
    return part._lib.hb2_batch_branch_component_likelihoods(part._h, 0, len(po), ppo, int(K), pbk, pv, pw, None, ppi, ps, pr)


def test_refusals_leave_partition_usable():
    w, _ = gc.load("mg94_8x60_c1")
    rng = np.random.default_rng(26)
    branch_k, V, W, _ = meme_sets(w, 2, 8, rng)
    pats = rng.choice(w.S, 8, replace=False)
    lf = LF(w)
    lf.set_all_matrices()
    lnl = lf.compute()
    good = lf.part.batch_branch_component_likelihoods(pats, V, W, w.pi, branch_k=branch_k)
    R = W.shape[1]
    bad_k, bad_pat = branch_k.copy(), pats.copy()
    bad_k[0] = 3
    bad_pat[2] = w.S
    cases = [((pats, 0, branch_k, V, W, w.pi), "K=0 outside 1..4"), ((pats, 5, branch_k, V, W, w.pi), "K=5 outside 1..4"),
             ((pats, 2, bad_k, V, W, w.pi), r"branchK\[0\]=3 outside 1..2"),
             ((pats, 2, branch_k, V, None, w.pi), "weights must not be null .with one row per branch every row would equal siteLnL"),
             ((pats, 2, branch_k, None, W, w.pi), "null argument"), ((pats, 2, branch_k, V, W, None), "null argument"),
             ((bad_pat, 2, branch_k, V, W, w.pi), rf"patternOf\[2\]={w.S} out of range")]
    for args, msg in cases:
        site, rows = np.full(8, 7.0), np.full((8, R), 7.0)
        assert _raw(lf.part, *args, site, rows) != 0
        assert re.search(msg, lf.part._lib.hb2_last_error().decode()), lf.part._lib.hb2_last_error()
        assert np.all(site == 7.0) and np.all(rows == 7.0)
    assert _raw(lf.part, pats, 2, branch_k, V, W, w.pi, np.empty(8), None) != 0
    assert "rowLnL must not be null" in lf.part._lib.hb2_last_error().decode()
    # siteLnL is nullable
    rows = np.empty((8, R))
    _check(_raw(lf.part, pats, 2, branch_k, V, W, w.pi, None, rows))
    assert np.array_equal(rows, good[1])
    # nSets == 0 does nothing
    _check(_raw(lf.part, pats[:0], 2, branch_k, V[:0], W[:0], w.pi, np.empty(0), np.empty((0, R))))
    again = lf.part.batch_branch_component_likelihoods(pats, V, W, w.pi, branch_k=branch_k)
    assert np.array_equal(again[0], good[0]) and np.array_equal(again[1], good[1])
    assert lf.compute() == lnl
    lf.close()
    # 20 states: refused like the other batch entry points, and the partition still evaluates
    w20 = tree_workload(flat_tree(star(5)), 20, 40)
    lf = LikelihoodFunction(w20, flags=engine.FLAG_FORCE_FP64)
    lf.set_all_matrices()
    lnl = lf.compute()
    nb = w20.tree.n_branches
    assert _raw(lf.part, [0], 1, None, np.zeros((1, nb, 4)), np.ones((1, nb)), w20.pi, np.empty(1), np.empty((1, nb))) != 0
    assert "33..64-state" in lf.part._lib.hb2_last_error().decode()
    assert lf.compute() == lnl
    lf.close()
