"""GPU suite (pytest -m gpu): the CUDA path, called through the C ABI, against the oracle and the reference's
golden vectors.  north_star's contract is |dlnL| < 1e-6*|lnL|.  Two precisions are exercised:
  fp64 : HB2_FLAG_FORCE_FP64 -- fp64 kernels everywhere, held to 1e-10 (parity reference on the device)
  tc   : default flags -- 33..64-state models run on the tensor cores (wgmma, error-compensated 3xTF32 + anchors, fp32 conditionals),
         held to 1e-7 (10x inside the contract); other state counts use the fp64 register kernels in both modes.
Measured errors are appended to gpurun_out/parity_errors.jsonl for DESIGN.md."""
import json
import os

import numpy as np
import pytest

from hyphy_b200 import synth, LikelihoodFunction, engine
from oracle import port
from tests import golden_cases as gc

pytestmark = pytest.mark.gpu

RTOL_CONTRACT = 1e-6
MODES = {"fp64": (engine.FLAG_FORCE_FP64, 1e-10, 1e-8),     # flags, lnL rtol required, per-site atol
         "tc": (engine.FLAG_DEFAULT, 1e-7, 1e-5)}
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module", autouse=True)
def _need_gpu(engine_lib):
    assert engine.device_count() > 0, "GPU tests need a CUDA device (no fallback exists)"


@pytest.fixture(params=list(MODES))
def mode(request):
    return request.param


def LF(w, mode):
    return LikelihoodFunction(w, flags=MODES[mode][0])


def tol(w, mode):
    """(lnL rtol, per-site atol): only 33..64-state models take the tensor path."""
    if mode == "tc" and w.D > 32:
        return MODES["tc"][1], MODES["tc"][2]
    return MODES["fp64"][1], MODES["fp64"][2]


def record(test, name, mode, got, ref, site_err=None):
    try:
        os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
        with open(os.path.join(ROOT, "gpurun_out", "parity_errors.jsonl"), "a") as f:
            f.write(json.dumps({"test": test, "case": name, "mode": mode, "lnL": got, "ref": ref,
                                "rel": abs(got - ref) / abs(ref), "signed": (got - ref) / abs(ref),
                                "max_site_abs": site_err}) + "\n")
    except OSError:
        pass


def _site_lnl(sl, ss):
    return np.log(sl) - 64.0 * np.log(2.0) * ss


@pytest.mark.parametrize("name", gc.SMALL + gc.MEDIUM + gc.FULL)
def test_lnl_matches_reference_golden(name, mode):
    w, g = gc.load(name)
    lf = LF(w, mode)
    assert lf.part.precision_mode == (1 if (mode == "tc" and w.D > 32) else 0)
    lf.set_all_matrices()
    lnl, sl, ss = lf.compute(want_sites=True)
    lf.close()
    site = _site_lnl(sl, ss)
    err = float(np.abs(site[w.site_to_pattern] - g["site_lnL"]).max())
    record("golden", name, mode, lnl, g["lnL"], err)
    rtol, atol = tol(w, mode)
    assert abs(lnl - g["lnL"]) <= rtol * abs(g["lnL"]), (lnl, g["lnL"])
    assert err <= atol
    # a checksum of checksums: frequency-weighted per-pattern values must re-add to lnL
    assert abs((site * w.pattern_freq).sum() - lnl) <= 1e-9 * abs(lnl)
    assert np.all(sl > 0) and np.all(sl <= 1.0)


@pytest.mark.parametrize("name", ["c1_hky85_8x500", "nuc_300x200_scaling"])
def test_nucleotide_one_and_two_patterns_per_thread_agree_bitwise(name, monkeypatch):
    """4 states: prune_small_walk_kernel (one pattern per thread) and prune_small_walk_ilp_kernel (two) do the same arithmetic
    per pattern -- identical per-pattern values, both equal to the reference's; partial updates and pinned nodes included."""
    w, g = gc.load(name)
    L, I = w.tree.n_leaves, w.tree.n_internal
    rng = np.random.default_rng(11)
    fs = rng.integers(0, w.D, size=w.S)
    out = {}
    for ilp in ("1", "2"):
        monkeypatch.setenv("HB2_SMALL_ILP", ilp)
        lf = LF(w, "fp64")
        lf.set_all_matrices()
        lnl, sl, ss = lf.compute(want_sites=True)
        part = lf.compute(update_nodes=[2, L + 1])
        forced = lf.part.evaluate_forced(w.C - 1, w.pi, L + I // 2, fs)
        after = lf.compute(update_nodes=None)
        lf.close()
        out[ilp] = (lnl, sl, ss, part, forced, after)
        site = _site_lnl(sl, ss)
        assert abs(lnl - g["lnL"]) <= 1e-10 * abs(g["lnL"])
        assert float(np.abs(site[w.site_to_pattern] - g["site_lnL"]).max()) <= 1e-8
        assert part == lnl and after == lnl
    a, b = out["1"], out["2"]
    assert a[0] == b[0] and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])
    assert a[4][0] == b[4][0] and np.array_equal(a[4][1], b[4][1]) and np.array_equal(a[4][2], b[4][2])


def test_reference_own_golden_smallcodon(mode):
    """The reference's own golden vector: tests/hbltests/SimpleOptimizations/SmallCodon.bf:37 (-3189.516375 +- 0.002),
    evaluated at the parameters the reference binary fitted."""
    w, Qt, g = gc.load_smallcodon()
    lf = LF(w, mode)
    lf.set_all_matrices(Qt)
    lnl = lf.compute()
    lf.close()
    record("smallcodon", "SmallCodon.bf", mode, lnl, g["lnL_reference_run"])
    assert abs(lnl - g["lnL_reference_run"]) <= tol(w, mode)[0] * abs(lnl)
    assert abs(lnl - g["lnL_golden"]) < 0.002


@pytest.mark.parametrize("name", ["mg94_8x60_c4_ambig", "c1_hky85_8x500", "mg94_200x64_c4_scaling"])
def test_per_class_compute_block_matches_oracle(name, mode):
    """ComputeBlock semantics: one rate class at a time with (L, scaler count) outputs, combined on the host the
    way PopulateConditionalProbabilities does (likefunc2.cpp:828-859) == fused device path == oracle."""
    w, g = gc.load(name)
    rtol, atol = tol(w, mode)
    lf = LF(w, mode)
    lf.set_all_matrices()
    per_class = []
    for c in range(w.C):
        lnl_c, sl, ss = lf.compute_block(c, want_sites=True)
        P = np.stack([port.expm(w.Q_classes[c] * w.tree.t[b], w.D > 20) for b in range(w.tree.n_branches)])
        oL, oS = port.prune(w, P)
        np.testing.assert_allclose(_site_lnl(sl, ss), _site_lnl(oL, oS), rtol=0, atol=atol)
        assert abs(lnl_c - (w.pattern_freq * _site_lnl(oL, oS)).sum()) <= rtol * abs(lnl_c)
        per_class.append(np.log(w.class_weights[c]) + _site_lnl(sl, ss))
    fused = lf.compute()
    lf.close()
    host_combined = (w.pattern_freq * np.logaddexp.reduce(np.stack(per_class), axis=0)).sum()
    assert abs(fused - host_combined) <= 1e-10 * abs(fused)
    assert abs(fused - g["lnL"]) <= rtol * abs(g["lnL"])


def test_expm_matches_oracle():
    w, _ = gc.load("mg94_30x100_c4_ambig")
    lf = LF(w, "fp64")
    lf.set_all_matrices()
    for c in (0, 3):
        for b in (0, 7, w.tree.n_branches - 1):
            P = lf.part.read_transition(c, b)
            Po = port.expm(w.Q_classes[c] * w.tree.t[b], True)
            np.testing.assert_allclose(P, Po, rtol=0, atol=2e-14)
            np.testing.assert_allclose(P.sum(axis=1), 1.0, atol=1e-14)
    lf.close()


def test_expm_large_rates_and_zero():
    """Long branches need several squarings; a zero matrix must give the identity."""
    w = synth.codon_workload(6, 20, 1, seed=3)
    lf = LF(w, "fp64")
    Q = w.Q_classes[0]
    ts = np.array([0.0, 1e-6, 0.3, 2.0, 25.0, 400.0, 3.0, 0.01, 1.0])[: w.tree.n_branches]
    lf.part.set_matrices(0, np.arange(len(ts)), Q[None] * ts[:, None, None])
    for b, t in enumerate(ts):
        P = lf.part.read_transition(0, b)
        np.testing.assert_allclose(P, port.expm(Q * t, True), rtol=0, atol=5e-13 if t < 5 else 1e-10)
    np.testing.assert_array_equal(lf.part.read_transition(0, 0), np.eye(61))
    np.testing.assert_allclose(lf.part.read_transition(0, 5), np.tile(w.pi, (61, 1)), atol=1e-9)
    lf.close()


def test_expm_shared_powers_and_fallbacks():
    """The shared-powers path (one power table per rate class, a scalar polynomial per branch) against the oracle, together
    with everything that must NOT take it: a branch whose matrix is not a multiple of the class's reference direction,
    very long branches (squarings), later single-matrix batches judged against the CACHED direction, and both hand-over
    forms.  HB2_EXPM_SHARED=0 (the product kernel for every matrix) must give the same matrices to rounding."""
    w, _ = gc.load("mg94_30x100_c4_ambig")
    nb = w.tree.n_branches
    Qt = w.Qt()
    odd = synth.mg94_rev_Q(7.5) * 0.11                      # a different direction (another omega)
    Qt[1, 5] = odd
    Qt[2, 9] *= 60.0                                         # rho ~ 10: several squarings after the polynomial
    Qt[3, 11] *= 1e-7                                        # tiny rho
    Qt[0, 3] *= 0.0                                          # zero matrix -> identity

    def check(part, c, b, M, tol=3e-14):
        P = part.read_transition(c, b)
        Po = port.expm(M, True)
        np.testing.assert_allclose(P, Po, rtol=0, atol=tol)
        assert np.all(P >= 0) and np.abs(P.sum(axis=1) - 1.0).max() <= 1e-14

    lf = LF(w, "fp64")
    lf.set_all_matrices(Qt)
    for c in range(w.C):
        for b in (0, 3, 5, 9, 11, nb - 1):
            check(lf.part, c, b, Qt[c, b], 5e-13 if (c, b) == (2, 9) else 3e-14)
    np.testing.assert_array_equal(lf.part.read_transition(0, 3), np.eye(61))
    # single-matrix batches: proportional to the cached direction (polynomial, no products) and not proportional (products)
    lf.part.set_matrices(0, [7], Qt[0, 7][None] * 1.75)
    lf.part.set_matrices(1, [7], odd[None] * 0.5)
    check(lf.part, 0, 7, Qt[0, 7] * 1.75)
    check(lf.part, 1, 7, odd * 0.5)
    lnl_shared = lf.compute()
    # compiled hand-over: same matrices assembled on the device, class 2 moved to another direction afterwards
    lf.set_template()
    vals = w.compiled_values()
    lf.set_all_compiled(vals)
    for c in (0, 3):
        for b in (1, nb - 2):
            check(lf.part, c, b, w.Qt()[c, b])
    lf.part.set_matrices_compiled(2, [4], vals[2, 4][None] * 3.0)
    check(lf.part, 2, 4, w.Qt()[2, 4] * 3.0)
    skew = vals[2, 6].copy()
    skew[::3] *= 1.3                                         # not a multiple any more
    lf.part.set_matrices_compiled(2, [6], skew[None])
    ei, ef, nf, cf = w.compiled_template()
    M = np.zeros((61, 61))
    M.flat[ei] = skew[ef]
    M[np.diag_indices(61)] = -M.sum(axis=1)
    check(lf.part, 2, 6, M)
    lf.close()
    os.environ["HB2_EXPM_SHARED"] = "0"
    try:
        lf = LF(w, "fp64")
        lf.set_all_matrices(Qt)
        lf.part.set_matrices(0, [7], Qt[0, 7][None] * 1.75)
        lf.part.set_matrices(1, [7], odd[None] * 0.5)
        lnl_products = lf.compute()
        lf.close()
    finally:
        del os.environ["HB2_EXPM_SHARED"]
    assert abs(lnl_shared - lnl_products) <= 1e-12 * abs(lnl_products)


def test_host_transition_matrices_path(mode):
    """HB2_MATRIX_TRANS: host-exponentiated P (GetCompExp()->theData) gives the same lnL."""
    w, g = gc.load("mg94_8x60_c1")
    lf = LF(w, mode)
    P = np.stack([port.expm(w.Q_classes[0] * w.tree.t[b], True) for b in range(w.tree.n_branches)])
    lf.part.set_matrices_ptrs(0, lf.all_nodes, list(P), engine.MATRIX_TRANS)
    lnl = lf.compute()
    lf.close()
    assert abs(lnl - g["lnL"]) <= max(tol(w, mode)[0], 1e-12) * abs(g["lnL"])


@pytest.mark.parametrize("name", ["mg94_30x100_c4_ambig", "c1_hky85_8x500"])
def test_compiled_template_equals_dense_matrices(name, mode):
    """hb2_set_rate_template + hb2_set_matrices_compiled (the reference's _CompiledMatrixData hand-over, incl. the
    MultByFreqs column multiplier for HKY85) must give the matrices and lnL of the dense hand-over."""
    w, g = gc.load(name)
    lf = LF(w, mode)
    lf.set_all_matrices()
    dense = lf.compute()
    Pd = lf.part.read_transition(w.C - 1, 4)
    lf.close()
    lf = LF(w, mode)
    lf.set_template()
    lf.set_all_compiled()
    comp = lf.compute()
    np.testing.assert_allclose(lf.part.read_transition(w.C - 1, 4), Pd, rtol=0, atol=1e-14)
    # partial update through the compiled path
    w.tree.t[2] *= 1.3
    V = w.compiled_values()
    for c in range(w.C):
        lf.part.set_matrices_compiled(c, [2], V[c, 2:3])
    upd = lf.compute(update_nodes=[2])
    ref, _ = port.lnl(w)
    w.tree.t[2] /= 1.3
    lf.close()
    assert abs(comp - dense) <= 1e-12 * abs(dense)
    assert abs(upd - ref) <= tol(w, mode)[0] * abs(ref)
    with pytest.raises(engine.EngineError, match="hb2_set_rate_template"):
        lf2 = LF(w, mode)
        try:
            lf2.part.n_formulas = 3
            lf2.part.set_matrices_compiled(0, [0], np.zeros((1, 3)))
        finally:
            lf2.close()


def test_partial_update_equals_full_recompute(mode):
    """DetermineNodesForUpdate semantics (tree.cpp:3117): change one branch, pass only that node; the engine must
    re-prune its ancestors and reuse every other cached conditional."""
    w, _ = gc.load("mg94_30x100_c4_ambig")
    rtol, _ = tol(w, mode)
    lf = LF(w, mode)
    lf.set_all_matrices()
    base = lf.compute()
    for node in [0, 5, w.tree.n_leaves + 2, w.tree.n_branches - 1]:
        w.tree.t[node] *= 1.7
        Qt = w.Qt()
        for c in range(w.C):
            lf.part.set_matrices(c, [node], Qt[c, node:node + 1])
        got = lf.compute(update_nodes=[node])
        ref, _ = port.lnl(w)
        assert abs(got - ref) <= rtol * abs(ref)
        assert got != base
    # idempotence: nothing changed, empty update list -> same value; a forced full recompute agrees (bit for bit on the
    # fp64 path; the walk kernel may fold a node's children in a different order, i.e. fp32 rounding noise)
    again = lf.compute(update_nodes=[])
    full = lf.compute(update_nodes=None)
    assert again == got
    assert full == got if (mode == "fp64" or w.D <= 32) else abs(full - got) <= 1e-8 * abs(got)
    lf.close()
    gc._cache.pop("mg94_30x100_c4_ambig", None)          # this test edited the cached workload's branch lengths


def test_root_frequencies_and_weights_only_change(mode):
    w, _ = gc.load("mg94_8x60_c4_ambig")
    lf = LF(w, mode)
    lf.set_all_matrices()
    lf.compute()
    w2 = np.array([0.1, 0.2, 0.3, 0.4])
    got = lf.compute(update_nodes=[], weights=w2)
    ref, _ = port.lnl(w, weights=w2)
    lf.close()
    assert abs(got - ref) <= tol(w, mode)[0] * abs(ref)


def test_mixture_matrices_bsrel(mode):
    """Explicit-form models P = sum_k w_k Exp(Q_k) per branch (tree.cpp:3047-3089)."""
    w = synth.codon_workload(10, 40, 1, seed=11)
    K = 3
    comps = [synth.mg94_rev_Q(om) for om in (0.1, 1.0, 4.0)]
    wk = np.array([0.6, 0.3, 0.1])
    nb = w.tree.n_branches
    M = np.stack([np.stack([Qk * w.tree.t[b] for Qk in comps]) for b in range(nb)])      # [nb, K, D, D]
    lf = LF(w, mode)
    lf.part.set_mixture_matrices(0, np.arange(nb), M, np.tile(wk, (nb, 1)))
    got = lf.compute()
    P = np.stack([sum(wk[k] * port.expm(M[b, k], True) for k in range(K)) for b in range(nb)])
    oL, oS = port.prune(w, P)
    ref = (w.pattern_freq * _site_lnl(oL, oS)).sum()
    np.testing.assert_allclose(lf.part.read_transition(0, 3), P[3], atol=1e-14)
    lf.close()
    assert abs(got - ref) <= tol(w, mode)[0] * abs(ref)


@pytest.mark.parametrize("name", gc.MIXTURE_SMALL + gc.MIXTURE_FULL)
def test_mixture_model_matches_reference_golden(name, mode):
    """BASELINE.json configs[2] (c3: BUSTED shape, 100 taxa x 1500 codons, K = 3 explicit-form mixture on every branch)
    and a small sibling, through hb2_set_mixture_matrices, against the unmodified reference binary's output."""
    w, g = gc.load(name)
    rtol, atol = tol(w, mode)
    M, wk = w.mixture_Qt()
    lf = LF(w, mode)
    lf.part.set_mixture_matrices(0, np.arange(w.tree.n_branches), M, wk)
    lnl, sl, ss = lf.compute(want_sites=True)
    err = float(np.abs(_site_lnl(sl, ss)[w.site_to_pattern] - g["site_lnL"]).max())
    record("golden_mixture", name, mode, lnl, g["lnL"], err)
    # second evaluation with every component changed, then back: the mixture path is re-entrant and leaves no residue
    M2, _ = w.mixture_Qt(perturb=0.25)
    lf.part.set_mixture_matrices(0, np.arange(w.tree.n_branches), M2, wk)
    other = lf.compute()
    lf.part.set_mixture_matrices(0, np.arange(w.tree.n_branches), M, wk)
    again = lf.compute()
    lf.close()
    assert abs(lnl - g["lnL"]) <= rtol * abs(g["lnL"])
    assert err <= atol
    assert other != lnl and again == lnl


@pytest.mark.parametrize("name", gc.HUGE)
def test_c5_absrel_size_matches_reference_golden(name, mode):
    """BASELINE.json configs[4] (c5: 500 taxa x 5000 codons x 4 classes; 5.2 GB of fp32 conditionals, 10.4 GB in fp64)
    on ONE GPU against the unmodified reference binary's lnL and per-site log-likelihoods."""
    w, g = gc.load(name)
    rtol, atol = tol(w, mode)
    lf = LF(w, mode)
    lf.set_template()
    lf.set_all_compiled()
    lnl, sl, ss = lf.compute(want_sites=True)
    err = float(np.abs(_site_lnl(sl, ss)[w.site_to_pattern] - g["site_lnL"]).max())
    record("golden_c5", name, mode, lnl, g["lnL"], err)
    lf.close()
    assert abs(lnl - g["lnL"]) <= rtol * abs(g["lnL"])
    assert err <= atol


def test_plain_matrices_then_mixtures_before_first_evaluate(mode):
    """The usual BS-REL sequence: plain matrices for most branches, mixtures for a few, no evaluation in between.  The
    mixture hand-over must not disturb plain matrices whose H2D copy is still in flight (ADVICE r1: staging race)."""
    w = synth.codon_workload(14, 48, 1, seed=5)
    nb = w.tree.n_branches
    Qt = w.Qt()
    comps = [synth.mg94_rev_Q(om) for om in (0.2, 1.0, 3.0)]
    wk = np.array([0.5, 0.4, 0.1])
    mixed = np.array([1, 4, 9, nb - 1])
    M = np.stack([np.stack([Qk * w.tree.t[b] for Qk in comps]) for b in mixed])
    lf = LF(w, mode)
    lf.part.set_matrices(0, np.arange(nb), Qt[0])                 # every branch plain first (queued, not yet flushed)
    lf.part.set_mixture_matrices(0, mixed, M, np.tile(wk, (len(mixed), 1)))
    got = lf.compute()
    P = np.stack([port.expm(Qt[0, b], True) for b in range(nb)])
    for i, b in enumerate(mixed):
        P[b] = sum(wk[k] * port.expm(M[i, k], True) for k in range(3))
    oL, oS = port.prune(w, P)
    ref = (w.pattern_freq * _site_lnl(oL, oS)).sum()
    for b in (0, 1, 4, nb - 1):
        np.testing.assert_allclose(lf.part.read_transition(0, b), P[b], atol=5e-14)
    lf.close()
    assert abs(got - ref) <= tol(w, mode)[0] * abs(ref)


def test_same_slot_handed_over_twice_last_one_wins(mode):
    """A (class, node) slot staged twice before an evaluation -- dense/dense, compiled/dense, dense/compiled -- must end up
    holding the LAST matrix (SetCompExp semantics, calcnode.cpp:714), never a mix of the two (ADVICE r1)."""
    w, _ = gc.load("mg94_30x100_c4_ambig")
    nb = w.tree.n_branches
    good = w.Qt()
    bad = w.Qt(perturb=0.7)
    lf = LF(w, mode)
    lf.set_template()
    lf.set_all_matrices(good)
    ref = lf.compute()
    vals_good, vals_bad = w.compiled_values(), w.compiled_values(perturb=0.7)
    nodes = np.arange(nb)
    # dense(bad) then dense(good)
    for c in range(w.C):
        lf.part.set_matrices(c, nodes, bad[c])
        lf.part.set_matrices(c, nodes[::-1].copy(), good[c][::-1].copy())
    assert lf.compute() == ref
    # compiled(bad) then dense(good)
    for c in range(w.C):
        lf.part.set_matrices_compiled(c, nodes, vals_bad[c])
        lf.part.set_matrices(c, nodes, good[c])
    assert lf.compute() == ref
    # dense(bad) then compiled(good), then compiled(bad) then compiled(good) for half of the nodes
    for c in range(w.C):
        lf.part.set_matrices(c, nodes, bad[c])
        lf.part.set_matrices_compiled(c, nodes, vals_good[c])
    a = lf.compute()
    for c in range(w.C):
        lf.part.set_matrices_compiled(c, nodes[: nb // 2], vals_bad[c][: nb // 2])
        lf.part.set_matrices_compiled(c, nodes[: nb // 2], vals_good[c][: nb // 2])
    b = lf.compute()
    lf.close()
    assert a == b
    assert abs(a - ref) <= 1e-12 * abs(ref)          # compiled vs dense assembly differ by rounding only


@pytest.mark.parametrize("D,taxa,sites,C", [(20, 12, 300, 1), (20, 40, 200, 4), (2, 9, 64, 1), (16, 7, 100, 2), (29, 6, 50, 1), (62, 9, 70, 1)])
def test_other_state_counts(D, taxa, sites, C, mode):
    """Protein-sized (20), binary, dinucleotide (16) and non-61 codon tables (60-63 -> padded 64) state spaces."""
    w = synth.generic_workload(D, taxa, sites, C)
    lf = LF(w, mode)
    lf.set_all_matrices()
    got = lf.compute()
    lf.close()
    ref, _ = port.lnl(w, sparse_storage=False)
    record("states", w.name, mode, got, ref)
    assert abs(got - ref) <= tol(w, mode)[0] * abs(ref)


@pytest.mark.parametrize("D,taxa,sites,C", [(20, 24, 400, 2), (16, 11, 130, 1), (29, 10, 90, 2)])
def test_protein_sized_states_ambiguity_partial_forced_readback(D, taxa, sites, C):
    """16 / 24 / 32 padded states run on the FP64 tensor pipe (prune_small_dmma_kernel): ambiguous leaves, partial updates
    (bit-identical to a full recomputation), a pinned node against the oracle, and the conditionals' read-back."""
    w = synth.generic_workload(D, taxa, sites, C, seed=77)
    rng = np.random.default_rng(5)
    # make some leaf observations ambiguous: 7 random 0/1 vectors (the reference's resolution vectors, likefunc.cpp:4299)
    amb = (rng.random((7, D)) < 0.3).astype(float)
    amb[np.arange(7), rng.integers(0, D, 7)] = 1.0
    w.ambig = amb
    ls = w.leaf_states.copy()
    hit = rng.random(ls.shape) < 0.04
    ls[hit] = -(rng.integers(0, 7, size=hit.sum()) + 1)
    w.leaf_states = ls
    lf = LF(w, "fp64")
    assert lf.part.pruning_kernel == "prune_small_dmma_kernel"
    lf.set_all_matrices()
    got = lf.compute()
    ref, _ = port.lnl(w, sparse_storage=False)
    assert abs(got - ref) <= 1e-10 * abs(ref)
    L, I = w.tree.n_leaves, w.tree.n_internal
    # conditionals of every internal node, class 0
    P0 = np.stack([port.expm(w.Q_classes[0] * w.tree.t[b], False) for b in range(w.tree.n_branches)])
    _, _, ocond = port.prune(w, P0, want_cond=True)
    for inode in range(I):
        cond, e = lf.part.read_conditionals(0, inode)
        rowmax = ocond[inode].max(axis=1, keepdims=True)
        got = cond * np.exp2(e)[:, None]
        # the oracle stores conditionals the reference's way: multiplied by 2^64 whenever a row fell below 2^-64
        # (tree_evaluator.cpp:411-525); the engine's (mantissa, binary exponent) pair is the true value
        k = np.rint(np.log2(rowmax[:, 0] / got.max(axis=1)) / 64.0)
        assert np.all(k >= 0)
        got = got * np.exp2(64.0 * k)[:, None]
        err = np.abs(got - ocond[inode]) - (1e-12 * rowmax + 1e-9 * ocond[inode])
        bad = np.unravel_index(np.argmax(err), err.shape)
        assert err.max() <= 0, (inode, bad, cond[bad], int(e[bad[0]]), ocond[inode][bad], float(rowmax[bad[0], 0]), w.leaf_states[:, bad[0]].min())
        assert np.all(cond.max(axis=1) >= 0.5) and np.all(cond.max(axis=1) <= 1.0)
    # partial updates
    for node in [1, L + 1, w.tree.n_branches - 1]:
        w.tree.t[node] *= 1.4
        Qt = w.Qt()
        for c in range(w.C):
            lf.part.set_matrices(c, [node], Qt[c, node:node + 1])
        part = lf.compute(update_nodes=[node])
        ref, _ = port.lnl(w, sparse_storage=False)
        assert abs(part - ref) <= 1e-10 * abs(ref)
        assert lf.compute(update_nodes=None) == part
    # a pinned node: leaf, internal, root
    c = w.C - 1
    Qt = w.Qt()
    Pc = np.stack([port.expm(q, False) for q in Qt[c]])
    base, bl, bs = lf.compute_block(c, want_sites=True)
    children = w.tree.children()
    for node in (0, L + I // 2, L + I - 1):
        fs = rng.integers(0, D, size=w.S)
        oL, oS = port.prune_forced(w, Pc, node, fs)
        lnl, sl, ss = lf.part.evaluate_forced(c, w.pi, node, fs, update_nodes=[node] if node < L else children[node - L])
        ok = oL > 0
        assert np.array_equal(sl > 0, ok)
        assert np.abs(_site_lnl(np.maximum(sl, 1e-300), ss)[ok] - _site_lnl(np.maximum(oL, 1e-300), oS)[ok]).max() <= 1e-9
        again, al, as_ = lf.compute_block(c, update_nodes=[node] if node < L else children[node - L], want_sites=True)
        assert again == base and np.array_equal(al, bl) and np.array_equal(as_, bs)
    lf.close()


@pytest.mark.parametrize("name", ["mg94_8x60_c4_ambig", "mg94_200x64_c4_scaling", "c1_hky85_8x500"])
def test_forced_states_match_oracle(name, mode):
    """ComputeBlock(..., branchIndex, branchValues) -- one node pinned to a per-pattern state (tree_evaluator.cpp:3624,
    173-181, 585-592, 4059): leaf, internal node, root; full and partial (children-of-the-node) update lists; the
    caches must be usable again after the host-style recomputation of the touched path."""
    w, g = gc.load(name)
    rtol, atol = tol(w, mode)
    rng = np.random.default_rng(7)
    L, I = w.tree.n_leaves, w.tree.n_internal
    Qt = w.Qt()
    lf = LF(w, mode)
    lf.set_all_matrices(Qt)
    c = w.C - 1
    base, bl, bs = lf.compute_block(c, want_sites=True)
    P = np.stack([port.expm(q, w.D > 20) for q in Qt[c]])
    children = w.tree.children()
    for node in sorted({0, L - 1, L, L + I // 2, L + I - 1}):
        fs = rng.integers(0, w.D, size=w.S)
        oL, oS = port.prune_forced(w, P, node, fs)
        ref_site = _site_lnl(np.maximum(oL, 1e-300), oS)
        for upd in (None, [node] if node < L else children[node - L]):
            lnl, sl, ss = lf.part.evaluate_forced(c, w.pi, node, fs, update_nodes=upd)
            got_site = _site_lnl(np.maximum(sl, 1e-300), ss)
            ok = oL > 0
            assert np.array_equal(sl > 0, ok)
            assert np.abs(got_site[ok] - ref_site[ok]).max() <= max(atol, 1e-9), (node, upd is None)
            if ok.all():
                ref = (w.pattern_freq * ref_site).sum()
                assert abs(lnl - ref) <= rtol * abs(ref)
            else:
                assert lnl == -np.inf
        # what the host does next (AddBranchToForcedRecomputeList): recompute the touched path without forcing
        again, al, as_ = lf.compute_block(c, update_nodes=[node] if node < L else children[node - L], want_sites=True)
        if mode == "fp64" or w.D <= 32:
            assert again == base and np.array_equal(al, bl) and np.array_equal(as_, bs)
        else:           # tensor path: a partial plan multiplies the children in another order (fp32 rounding); no residue otherwise
            assert abs(again - base) <= 1e-8 * abs(base) and np.array_equal(as_, bs)
    # marginalisation identity on an internal node: sum over its states of the pinned likelihoods = the likelihood
    node = L + I // 3
    tot = np.zeros(w.S)
    for st in range(w.D):
        _, sl, ss = lf.part.evaluate_forced(c, w.pi, node, np.full(w.S, st), update_nodes=children[node - L])
        tot += sl * 2.0 ** (-64.0 * (ss - bs))
    lf.close()
    np.testing.assert_allclose(tot, bl, rtol=max(10 * atol, 1e-9))


def test_batched_site_likelihoods():
    """SURVEY 8f row 3 (FEL / MEME site phases): many one-pattern likelihoods with per-set matrices in one call.
    (a) every set = the model of the reference's fixture -> the reference's own per-site log-likelihoods;
    (b) per-set parameters (alpha-, beta-like scalings, two branch classes) -> the oracle, set by set."""
    w, g = gc.load("c2_mg94_50x1000_c1")
    nb = w.tree.n_branches
    lf = LF(w, "fp64")
    lf.set_template()
    vals = w.compiled_values()[0]                                  # [B, nF]
    pats = np.arange(w.S)
    got = lf.part.batch_site_likelihoods(pats, np.broadcast_to(vals, (w.S,) + vals.shape), w.pi)
    assert np.abs(got[w.site_to_pattern] - g["site_lnL"]).max() <= 1e-9
    assert abs((got * w.pattern_freq).sum() - g["lnL"]) <= 1e-10 * abs(g["lnL"])
    # (b) sets with their own synonymous / non-synonymous scalings on two classes of branches
    rng = np.random.default_rng(3)
    ei, ef, nf, cf = w.compiled_template()
    # which formulas are non-synonymous: the ones whose value moves with omega (the fixture's model has omega = 0.3)
    wq = synth.Workload(w.name, w.tree, w.D, w.pi, [synth.mg94_rev_Q(0.6)], w.class_weights, w.leaf_states, w.ambig, w.pattern_freq,
                        w.site_to_pattern, None, dict(w.meta, omegas=[0.6]))
    keys_nonsyn = ~np.isclose(wq.compiled_values()[0][0], vals[0])
    fg = np.zeros(nb, dtype=np.int64)
    fg[rng.choice(nb, nb // 3, replace=False)] = 1                  # "tested" branches
    n_sets = 40
    sets = rng.choice(w.S, n_sets, replace=False)
    alpha = rng.uniform(0.2, 3.0, n_sets)
    beta_bg = rng.uniform(0.0, 4.0, n_sets)
    beta_fg = rng.uniform(0.0, 12.0, n_sets)
    beta_fg[:5] = beta_bg[:5]                                       # a few sets whose two classes coincide
    V = np.empty((n_sets, nb, nf))
    for i in range(n_sets):
        for b in range(nb):
            V[i, b] = vals[b] * np.where(keys_nonsyn, (beta_fg[i] if fg[b] else beta_bg[i]) / 0.3, alpha[i])
    for bg in (fg, None):                                           # with the hint and without (same numbers either way)
        got = lf.part.batch_site_likelihoods(sets, V, w.pi, branch_group=bg)
        for i in range(n_sets):
            Qt = np.zeros((1, nb, 61, 61))
            for b in range(nb):
                M = np.zeros((61, 61))
                M.flat[ei] = V[i, b][ef]
                M[np.diag_indices(61)] = -M.sum(axis=1)
                Qt[0, b] = M
            w1 = synth.Workload("one", w.tree, w.D, w.pi, w.Q_classes, w.class_weights, w.leaf_states[:, sets[i]:sets[i] + 1], w.ambig,
                                np.array([1]), np.array([0]))
            ref, _ = port.lnl(w1, Qt=Qt)
            assert abs(got[i] - ref) <= 1e-10 * abs(ref) + 1e-12, (i, got[i], ref)
    lf.close()


def test_conditionals_readback_matches_oracle(mode):
    w, _ = gc.load("mg94_8x60_c1")
    lf = LF(w, mode)
    lf.set_all_matrices()
    lf.compute()
    P = np.stack([port.expm(w.Q_classes[0] * w.tree.t[b], True) for b in range(w.tree.n_branches)])
    _, _, ocond = port.prune(w, P, want_cond=True)
    for inode in range(w.tree.n_internal):
        cond, e = lf.part.read_conditionals(0, inode)
        # P entries carry ~1e-16 ABSOLUTE error (both here and in the reference), so tiny conditionals are compared
        # relative to the row maximum
        rowmax = ocond[inode].max(axis=1, keepdims=True)
        got = cond * np.exp2(e)[:, None]
        assert np.all(np.abs(got - ocond[inode]) <= (1e-12 if mode == "fp64" else 3e-6) * rowmax + (1e-9 if mode == "fp64" else 3e-5) * ocond[inode])
        assert np.all(cond.max(axis=1) >= 0.5) and np.all(cond.max(axis=1) <= 1.0)
    lf.close()


def test_impossible_pattern_gives_minus_infinity(mode):
    """tree_evaluator.cpp:4094-4112: a pattern with likelihood 0 makes the block -inf."""
    for w in (synth.nucleotide_workload(5, 30, seed=2), synth.codon_workload(5, 30, 1, seed=2)):
        lf = LF(w, mode)
        P = np.tile(np.eye(w.D), (w.tree.n_branches, 1, 1))     # zero-length branches: differing leaves are impossible
        lf.part.set_matrices(0, lf.all_nodes, P, engine.MATRIX_TRANS)
        assert lf.compute() == -np.inf
        lf.close()


def test_nan_is_propagated():
    w = synth.nucleotide_workload(5, 30, seed=2)
    lf = LF(w, "fp64")
    Qt = w.Qt()
    Qt[0, 2, 1, 1] = np.nan
    lf.set_all_matrices(Qt)
    assert np.isnan(lf.compute())
    lf.close()


def test_errors_are_reported_not_swallowed():
    w = synth.nucleotide_workload(5, 30, seed=2)
    lf = LF(w, "fp64")
    with pytest.raises(engine.EngineError, match="no matrix was ever set"):
        lf.compute()
    with pytest.raises(engine.EngineError):
        lf.part.set_matrices(0, [99], np.zeros((1, 4, 4)))
    lf.close()
    with pytest.raises(engine.EngineError, match="not supported"):
        engine.Partition(4, 70, 3, 1, 1, [0, 0, 0, -1], np.zeros((3, 4), dtype=np.int64), None, np.ones(4, dtype=np.int64))


def test_full_size_properties(mode):
    """At BASELINE.json's full size: golden lnL, linearity in pattern frequencies (doubling every frequency doubles
    lnL), and invariance under a permutation of the patterns."""
    w, g = gc.load("ns_mg94_200x2000_c4")
    rtol, _ = tol(w, mode)
    lf = LF(w, mode)
    lf.set_all_matrices()
    a = lf.compute()
    lf.close()
    assert abs(a - g["lnL"]) <= rtol * abs(g["lnL"])
    perm = np.random.default_rng(0).permutation(w.S)
    w2 = gc.CASES["ns_mg94_200x2000_c4"]()
    w2.leaf_states = np.ascontiguousarray(w.leaf_states[:, perm])
    w2.pattern_freq = w.pattern_freq[perm] * 2
    lf = LF(w2, mode)
    lf.set_all_matrices()
    b = lf.compute()
    lf.close()
    assert abs(b - 2 * a) <= 1e-11 * abs(b)


def test_more_class_tile_pairs_than_resident_ctas(mode):
    """12000 patterns x 4 classes = 376 (class, tile) pairs > 296 co-resident CTAs: the walk kernel must loop over pairs
    inside a CTA (K = 1 path); also exercises pattern padding (12000 is not a multiple of 128)."""
    w = synth.codon_workload(16, 12000, 4, seed=99, mean_t=0.4)
    assert w.S * w.C > 296 * 128
    lf = LF(w, mode)
    lf.set_template()
    lf.set_all_compiled()
    got, sl, ss = lf.compute(want_sites=True)
    lf.close()
    ref, site = port.lnl(w)
    record("bigS", w.name, mode, got, ref, float(np.abs(_site_lnl(sl, ss) - site).max()))
    assert abs(got - ref) <= tol(w, mode)[0] * abs(ref)
    assert np.abs(_site_lnl(sl, ss) - site).max() <= tol(w, mode)[1]


def test_tensor_path_against_fp64_path_deep_and_wide():
    """The tensor-core path against the fp64 kernels on the same device, on shapes chosen to stress error accumulation
    (500 taxa: ~1000 contractions per pattern) and short/long branch mixes.  Contract: 1e-6; required here: 1e-7."""
    for (taxa, codons, C, mean_t) in [(500, 96, 4, 0.05), (200, 128, 1, 0.005), (64, 256, 4, 0.3)]:
        w = synth.codon_workload(taxa, codons, C, seed=77, mean_t=mean_t)
        res = {}
        for m in ("fp64", "tc"):
            lf = LF(w, m)
            lf.set_all_matrices()
            res[m] = lf.compute(want_sites=True)
            lf.close()
        a, b = res["fp64"][0], res["tc"][0]
        site = np.abs(_site_lnl(res["fp64"][1], res["fp64"][2]) - _site_lnl(res["tc"][1], res["tc"][2])).max()
        record("tc_vs_fp64", w.name + f"_t{mean_t}", "tc", b, a, float(site))
        assert abs(a - b) <= 1e-7 * abs(a), (w.name, a, b)


def test_repeated_evaluations_are_bit_identical(mode):
    """Race hunt at full size: every CTA of the persistent walk kernel hands tiles to other CTAs through epoch flags and
    re-uses its shared-memory ring dozens of times per evaluation; a protocol slip shows up as a handful of patterns
    changing between identical evaluations (tools/stress_determinism.py is the long version of this test)."""
    w, _ = gc.load("ns_mg94_200x2000_c4")
    Qt = w.Qt()
    base = None
    for _ in range(3):
        lf = LF(w, mode)
        lf.set_all_matrices(Qt)
        for _ in range(10):
            lnl, site, scc = lf.compute(want_sites=True)
            if base is None:
                base = (lnl, site.copy(), scc.copy())
            assert lnl == base[0]
            assert np.array_equal(site, base[1]) and np.array_equal(scc, base[2])
        lf.close()


def _branch_nodes(w):
    """A leaf branch, the deepest internal branch, and a child of the root."""
    t = w.tree
    L, I = t.n_leaves, t.n_internal
    par = np.asarray(t.flat_parents)
    depth = np.zeros(L + I, dtype=int)
    for n in range(L + I - 2, -1, -1):               # parents have larger internal index: walk from the root down
        depth[n] = depth[L + par[n]] + 1
    internals = [n for n in range(L, L + I - 1)]
    deepest = max(internals, key=lambda n: depth[n])
    root_child = next(n for n in range(L + I - 1) if par[n] == I - 1)
    return sorted({0, int(np.argmax(depth[:L])), deepest, root_child})


@pytest.mark.parametrize("name", ["mg94_8x60_c4_ambig", "mg94_30x100_c4_ambig", "mg94_200x64_c4_scaling", "c1_hky85_8x500"])
def test_branch_cache_equals_full_evaluation(name, mode):
    """SURVEY 8f row 1: with only one branch's matrix changed, hb2_branch_cache_evaluate must return what a full
    evaluation with that matrix returns (all classes, per-pattern outputs included)."""
    w, g = gc.load(name)
    rtol, atol = tol(w, mode)
    Qt = w.Qt()
    lf = LF(w, mode)
    lf.set_all_matrices(Qt)
    base = lf.compute()
    for node in _branch_nodes(w):
        lf.part.branch_cache_build(node, w.pi)
        got0 = lf.part.branch_cache_evaluate(w.class_weights)
        assert abs(got0 - base) <= max(rtol, 1e-12) * abs(base)           # unchanged matrix: the same likelihood
        for scale in (0.3, 2.5):
            for c in range(w.C):
                lf.part.set_matrices(c, [node], (Qt[c, node] * scale)[None])
            got, sl, ss = lf.part.branch_cache_evaluate(w.class_weights, want_sites=True)
            Q2 = Qt.copy()
            Q2[:, node] *= scale
            ref_lf = LF(w, mode)
            ref_lf.set_all_matrices(Q2)
            ref, rl, rs = ref_lf.compute(want_sites=True)
            ref_lf.close()
            oracle_lnl, _ = port.lnl(w, Q2)
            record("branch_cache", f"{name}:node{node}:x{scale}", mode, got, oracle_lnl)
            assert abs(got - ref) <= max(rtol, 1e-12) * abs(ref), (node, scale, got, ref)
            assert abs(got - oracle_lnl) <= rtol * abs(oracle_lnl)
            assert np.abs(_site_lnl(sl, ss) - _site_lnl(rl, rs)).max() <= max(atol, 1e-9)
        for c in range(w.C):                                              # restore, caches stay consistent
            lf.part.set_matrices(c, [node], Qt[c, node][None])
        assert abs(lf.part.branch_cache_evaluate(w.class_weights) - base) <= max(rtol, 1e-12) * abs(base)
    # single-class form
    lf.part.branch_cache_build(0, w.pi)
    one = lf.part.branch_cache_evaluate(None, cat=w.C - 1)
    assert abs(one - lf.compute_block(w.C - 1)) <= max(rtol, 1e-12) * abs(one)
    lf.close()


def test_branch_cache_guards():
    w = synth.nucleotide_workload(6, 40, seed=3)
    lf = LF(w, "fp64")
    lf.set_all_matrices()
    with pytest.raises(engine.EngineError, match="never been evaluated"):
        lf.part.branch_cache_build(0, w.pi)
    lf.compute()
    with pytest.raises(engine.EngineError, match="no valid branch cache"):
        lf.part.branch_cache_evaluate(w.class_weights)
    lf.part.branch_cache_build(1, w.pi)
    lf.part.set_matrices(0, [2], w.Qt()[0, 2][None])
    with pytest.raises(engine.EngineError, match="a matrix of node 2 changed"):
        lf.part.branch_cache_evaluate(w.class_weights)
    lf.compute()                                             # a regular evaluation invalidates the cache
    with pytest.raises(engine.EngineError, match="no valid branch cache"):
        lf.part.branch_cache_evaluate(w.class_weights)
    # a matrix of another node that was already FLUSHED (read_transition flushes) must still be noticed (ADVICE r1)
    lf.part.branch_cache_build(1, w.pi)
    lf.part.set_matrices(0, [3], w.Qt()[0, 3][None] * 1.5)
    lf.part.read_transition(0, 3)
    with pytest.raises(engine.EngineError, match="a matrix of node 3 changed"):
        lf.part.branch_cache_evaluate(w.class_weights)
    lf.close()
