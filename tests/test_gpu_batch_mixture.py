"""GPU suite (pytest -m gpu): hb2_batch_site_mixture_likelihoods, batched one-pattern likelihoods whose branches carry
explicit-form mixtures P_b = sum_k w_k Exp(Q_k t_b) (MEME's site model, MEME.bf:381-386 and :656-680), against the
unmodified reference binary's per-site values, the oracle set by set, and the plain batch entry point."""
import numpy as np
import pytest

from hyphy_b200 import synth, LikelihoodFunction, engine
from hyphy_b200.engine import EngineError, _check, _d, _i, _dp
from oracle import port
from tests import golden_cases as gc
from tests.test_gpu_shapes import flat_tree, longdouble_sites, star, tree_workload, underflow_workload

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _need_gpu(engine_lib):
    assert engine.device_count() > 0, "GPU tests need a CUDA device (no fallback exists)"


def LF(w, flags=engine.FLAG_FORCE_FP64):
    lf = LikelihoodFunction(w, flags=flags)
    lf.set_template()
    return lf


def with_omegas(w, omegas):
    """The same codon workload whose model classes are MG94xREV at `omegas` (compiled_values then gives one row per omega)."""
    return synth.Workload(w.name, w.tree, w.D, w.pi, [synth.mg94_rev_Q(o) for o in omegas], np.full(len(omegas), 1.0 / len(omegas)),
                          w.leaf_states, w.ambig, w.pattern_freq, w.site_to_pattern, None, dict(w.meta, omegas=list(omegas)))


def one_pattern(w, p):
    return synth.Workload("one", w.tree, w.D, w.pi, w.Q_classes, w.class_weights, w.leaf_states[:, p:p + 1], w.ambig,
                          np.array([1]), np.array([0]))


def site_lnl(sl, ss):
    return np.log(sl) - 64.0 * np.log(2.0) * ss


def meme_sets(w, K, n_sets, rng):
    """MEME-shaped sets: a seeded third of the branches is tested (K components there, one elsewhere); every set draws
    its own alpha, beta_k and weights on the tested branches and a background beta.
    Returns (branch_k [B], formula values [n, R, nF], weights [n, R], tested [B])."""
    nb = w.tree.n_branches
    tested = np.zeros(nb, dtype=bool)
    tested[rng.choice(nb, max(1, nb // 3), replace=False)] = True
    branch_k = np.where(tested, K, 1).astype(np.int64)
    unit = with_omegas(w, [1.0]).compiled_values()[0]                    # [B, nF]: every formula at omega = 1
    nonsyn = ~np.isclose(with_omegas(w, [2.0]).compiled_values()[0][0], unit[0])
    R = int(branch_k.sum())
    V = np.empty((n_sets, R, unit.shape[1]))
    W = np.empty((n_sets, R))
    for i in range(n_sets):
        alpha, beta_bg = rng.uniform(0.2, 3.0), rng.uniform(0.0, 4.0)
        betas = np.sort(rng.uniform(0.0, 10.0, K))
        wk = rng.dirichlet(np.ones(K))
        r = 0
        for b in range(nb):
            for k in range(branch_k[b]):
                beta, wt = (betas[k], wk[k]) if tested[b] else (beta_bg, 1.0)
                V[i, r] = unit[b] * np.where(nonsyn, beta, alpha)
                W[i, r] = wt
                r += 1
    return branch_k, V, W, tested


def dense(w, v):
    """Rate matrix of one row of formula values (the template's scatter, diagonal = minus the row sum)."""
    ei, ef, _, _ = w.compiled_template()
    M = np.zeros((w.D, w.D))
    M.flat[ei] = v[ef]
    M[np.diag_indices(w.D)] = -M.sum(axis=1)
    return M


def oracle_set(w, pattern, branch_k, v, wt):
    """port.expm per row, the weighted sum in component order, port.prune on the one-pattern workload."""
    P = np.empty((w.tree.n_branches, w.D, w.D))
    r = 0
    for b in range(w.tree.n_branches):
        acc = None
        for _ in range(branch_k[b]):
            term = wt[r] * port.expm(dense(w, v[r]), True)
            acc = term if acc is None else acc + term
            r += 1
        P[b] = acc
    w1 = one_pattern(w, pattern)
    sl, ss = port.prune(w1, P)
    if sl[0] == 0.0:
        # the oracle, like the reference, boosts one node by at most ~2^495 (tree.cpp:129,182); the engine's exponent has
        # no such cap, so a wide node whose product falls further is held to the unscaled long-double recursion
        return float(longdouble_sites(w1, P)[0])
    return float(site_lnl(sl, ss)[0])


def plain_rows(branch_k, V, comp=0):
    """Plain (one matrix per branch) formula values made of component `comp` of every branch."""
    off = np.concatenate([[0], np.cumsum(branch_k)])
    return V[:, off[:-1] + np.minimum(comp, branch_k - 1)]


# ---------------------------------------------------------------------------------------------------------------------
# 1. the reference binary's own per-site values
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,n_pat", [("bsrel_12x80_k3", None), ("c3_bsrel_100x1500_k3", 256)])
def test_bsrel_fixture_matches_reference(name, n_pat):
    """Every set is the fixture's own K = 3 model: component rows from the compiled template at omega_k, the fixture's weights."""
    w, g = gc.load(name)
    mix = w.meta["mixture"]
    K, nb = len(mix["omegas"]), w.tree.n_branches
    comp = with_omegas(w, mix["omegas"]).compiled_values()                # [K, B, nF]
    rows = comp.transpose(1, 0, 2).reshape(nb * K, -1)                  # branch order, components consecutive
    pats = np.arange(w.S) if n_pat is None else np.sort(np.random.default_rng(5).choice(w.S, n_pat, replace=False))
    lf = LF(w)
    got = lf.part.batch_site_mixture_likelihoods(pats, np.broadcast_to(rows, (len(pats),) + rows.shape),
                                                 np.tile(mix["weights"], (len(pats), nb)), w.pi)
    lf.close()
    site = np.full(w.S, np.nan)
    site[pats] = got
    covered = np.isin(w.site_to_pattern, pats)
    assert covered.sum() >= len(pats)
    assert np.abs(site[w.site_to_pattern][covered] - g["site_lnL"][covered]).max() <= 1e-9
    if n_pat is None:
        assert abs((got * w.pattern_freq).sum() - g["lnL"]) <= 1e-10 * abs(g["lnL"])


# ---------------------------------------------------------------------------------------------------------------------
# 2. MEME-shaped sets against the oracle, set by set
# ---------------------------------------------------------------------------------------------------------------------
def _meme_workload(name):
    if name == "codon400_star":
        return underflow_workload("codon400"), 4
    w, _ = gc.load(name)
    return w, 12


@pytest.mark.parametrize("K", [2, 3])
@pytest.mark.parametrize("name", ["c2_mg94_50x1000_c1", "mg94_8x60_c4_ambig", "codon400_star"])
def test_meme_sets_match_oracle(name, K):
    w, n_sets = _meme_workload(name)
    rng = np.random.default_rng(100 * K + len(name))
    branch_k, V, W, tested = meme_sets(w, K, n_sets, rng)
    if len(w.ambig):                                                     # patterns with ambiguous leaves first
        amb = np.nonzero((w.leaf_states < 0).any(axis=0))[0]
        pats = np.concatenate([amb[:n_sets // 2], rng.choice(w.S, n_sets - min(len(amb), n_sets // 2), replace=False)])
        assert (w.leaf_states[:, pats] < 0).any()
    else:
        pats = rng.choice(w.S, n_sets, replace=False)
    ref = np.array([oracle_set(w, pats[i], branch_k, V[i], W[i]) for i in range(n_sets)])
    assert np.all(np.isfinite(ref))
    lf = LF(w)
    for bg in (tested.astype(np.int64), None):
        got = lf.part.batch_site_mixture_likelihoods(pats, V, W, w.pi, branch_k=branch_k, branch_group=bg)
        err = np.abs(got - ref)
        assert np.all(err <= 1e-10 * np.abs(ref) + 1e-12), (bg is None, err.max(), got, ref)
    lf.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3. degenerate forms
# ---------------------------------------------------------------------------------------------------------------------
def test_degenerate_forms():
    w, _ = gc.load("c2_mg94_50x1000_c1")
    rng = np.random.default_rng(7)
    branch_k, V, W, tested = meme_sets(w, 2, 24, rng)
    pats = rng.choice(w.S, 24, replace=False)
    bg = tested.astype(np.int64)
    lf = LF(w)
    # K = 1 with unit weights is the plain entry point, bit for bit
    P0 = plain_rows(branch_k, V)
    for hint in (bg, None):
        plain = lf.part.batch_site_likelihoods(pats, P0, w.pi, branch_group=hint)
        mixed = lf.part.batch_site_mixture_likelihoods(pats, P0, np.ones(P0.shape[:2]), w.pi, branch_group=hint)
        assert np.array_equal(plain, mixed)
    plain = lf.part.batch_site_likelihoods(pats, P0, w.pi, branch_group=bg)
    # the EBF shape: weights (1, 0) on every tested branch = the plain set made of component 0
    W10 = np.where(W == 1.0, 1.0, 0.0)
    off = np.concatenate([[0], np.cumsum(branch_k)])
    W10[:, off[:-1][tested]] = 1.0
    got = lf.part.batch_site_mixture_likelihoods(pats, V, W10, w.pi, branch_k=branch_k, branch_group=bg)
    assert np.all(np.abs(got - plain) <= 1e-13 * np.abs(plain))
    # two identical components weighted (0.3, 0.7) = the single component
    V2 = V.copy()
    V2[:, off[:-1][tested] + 1] = V2[:, off[:-1][tested]]
    W37 = np.ones_like(W)
    W37[:, off[:-1][tested]], W37[:, off[:-1][tested] + 1] = 0.3, 0.7
    got = lf.part.batch_site_mixture_likelihoods(pats, V2, W37, w.pi, branch_k=branch_k, branch_group=bg)
    assert np.all(np.abs(got - plain) <= 1e-13 * np.abs(plain))
    lf.close()


# ---------------------------------------------------------------------------------------------------------------------
# 4. chunking
# ---------------------------------------------------------------------------------------------------------------------
def test_chunks_match_small_calls():
    """More than 1024 sets (the chunk cap) in one call = the same sets in small separate calls, bit for bit."""
    w, _ = gc.load("mg94_8x60_c1")
    rng = np.random.default_rng(8)
    n = 1100
    branch_k, V, W, tested = meme_sets(w, 2, n, rng)
    pats = rng.integers(0, w.S, n)
    lf = LF(w)
    whole = lf.part.batch_site_mixture_likelihoods(pats, V, W, w.pi, branch_k=branch_k)
    parts = np.concatenate([lf.part.batch_site_mixture_likelihoods(pats[s:s + 100], V[s:s + 100], W[s:s + 100], w.pi, branch_k=branch_k)
                            for s in range(0, n, 100)])
    lf.close()
    assert np.all(np.isfinite(whole))
    assert np.array_equal(whole, parts)


# ---------------------------------------------------------------------------------------------------------------------
# 5. isolation and re-entry
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("flags", [engine.FLAG_FORCE_FP64, engine.FLAG_DEFAULT])
def test_resident_state_untouched(flags):
    w, _ = gc.load("mg94_8x60_c4_ambig")
    rng = np.random.default_rng(9)
    lf = LF(w, flags)
    lf.set_all_matrices()
    before = lf.compute()
    fel_k, fel_V, _, _ = meme_sets(w, 1, 30, rng)
    pats = rng.choice(w.S, 30, replace=False)
    fel = lf.part.batch_site_likelihoods(pats, fel_V, w.pi)
    branch_k, V, W, _ = meme_sets(w, 3, 40, rng)                      # more rows per set: the batch buffers grow
    lf.part.batch_site_mixture_likelihoods(rng.choice(w.S, 40), V, W, w.pi, branch_k=branch_k)
    assert lf.compute() == before
    assert np.array_equal(lf.part.batch_site_likelihoods(pats, fel_V, w.pi), fel)
    lf.close()


# ---------------------------------------------------------------------------------------------------------------------
# 6. values and guards
# ---------------------------------------------------------------------------------------------------------------------
def test_zero_formula_values_give_identity():
    w, _ = gc.load("mg94_8x60_c1")
    rng = np.random.default_rng(10)
    branch_k, V, W, _ = meme_sets(w, 2, w.S, rng)
    lf = LF(w)
    got = lf.part.batch_site_mixture_likelihoods(np.arange(w.S), np.zeros_like(V), W, w.pi, branch_k=branch_k)
    lf.close()
    const = np.all(w.leaf_states == w.leaf_states[:1], axis=0) & (w.leaf_states[0] >= 0)
    assert const.any() and (~const).any()
    assert np.all(got[~const] == -np.inf)
    np.testing.assert_allclose(got[const], np.log(w.pi[w.leaf_states[0, const]]), rtol=1e-12)


def test_nan_weight_stays_in_its_set():
    w, _ = gc.load("mg94_8x60_c1")
    rng = np.random.default_rng(12)
    branch_k, V, W, tested = meme_sets(w, 2, 16, rng)
    pats = rng.choice(w.S, 16, replace=False)
    lf = LF(w)
    clean = lf.part.batch_site_mixture_likelihoods(pats, V, W, w.pi, branch_k=branch_k)
    Wn = W.copy()
    Wn[5, int(np.concatenate([[0], np.cumsum(branch_k)])[np.nonzero(tested)[0][0]])] = np.nan
    got = lf.part.batch_site_mixture_likelihoods(pats, V, Wn, w.pi, branch_k=branch_k)
    lf.close()
    assert np.isnan(got[5])
    others = np.arange(16) != 5
    assert np.array_equal(got[others], clean[others])


def _raw(part, pats, K, branch_k, V, W, root):
    """The C entry point with arguments the Python wrapper would not let through."""
    po, ppo = _i(pats)
    pbk = None if branch_k is None else _i(branch_k)[1]
    v, pv = (None, None) if V is None else _d(V)
    wt, pw = (None, None) if W is None else _d(W)
    pi, ppi = _d(root)
    out = np.empty(len(po))
    _check(part._lib.hb2_batch_site_mixture_likelihoods(part._h, 0, len(po), ppo, int(K), pbk, pv, pw, None, ppi, out.ctypes.data_as(_dp)))
    return out


def test_refusals_leave_partition_usable():
    w, _ = gc.load("mg94_8x60_c1")
    rng = np.random.default_rng(13)
    branch_k, V, W, _ = meme_sets(w, 2, 8, rng)
    pats = rng.choice(w.S, 8, replace=False)
    lf = LF(w)
    lf.set_all_matrices()
    lnl = lf.compute()
    good = lf.part.batch_site_mixture_likelihoods(pats, V, W, w.pi, branch_k=branch_k)
    bad_k = branch_k.copy()
    bad_k[0] = 3
    zero_k = branch_k.copy()
    zero_k[1] = 0
    cases = [((0, branch_k, V, W), "K=0 outside 1..4"), ((5, branch_k, V, W), "K=5 outside 1..4"),
             ((2, bad_k, V, W), r"branchK\[0\]=3 outside 1..2"), ((2, zero_k, V, W), r"branchK\[1\]=0 outside 1..2"),
             ((2, branch_k, V, None), "weights must not be null"), ((2, branch_k, None, W), "formulaValues must not be null")]
    for (K, bk, v, wt), msg in cases:
        with pytest.raises(EngineError, match=msg):
            _raw(lf.part, pats, K, bk, v, wt, w.pi)
        assert np.array_equal(_raw(lf.part, pats, 2, branch_k, V, W, w.pi), good)
        assert lf.compute() == lnl
    lf.close()
    # 20 states: refused like the plain entry point, and the partition still evaluates
    w20 = tree_workload(flat_tree(star(5)), 20, 40)
    lf = LikelihoodFunction(w20, flags=engine.FLAG_FORCE_FP64)
    lf.set_all_matrices()
    lnl = lf.compute()
    nb = w20.tree.n_branches
    with pytest.raises(EngineError, match="33..64-state"):
        _raw(lf.part, [0], 1, None, np.zeros((1, nb, 4)), np.ones((1, nb)), w20.pi)
    assert lf.compute() == lnl
    ref, _ = port.lnl(w20)
    assert abs(lnl - ref) <= 1e-10 * abs(ref)
    lf.close()
