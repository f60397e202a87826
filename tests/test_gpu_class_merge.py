"""GPU suite (pytest -m gpu): the rate-class merge L_s = sum_c w_c L_{c,s} at its edges -- weights of 0 and tiny weights on
the class that sits highest, classes thousands of bits apart, impossible patterns, NaN, many classes -- against the exact
reference of tests/class_merge_cases.py (pinned on the CPU by tests/test_class_merge_reference.py).

Each case is checked twice:
  (A) the engine's own per-class outputs (hb2_evaluate of every class) merged exactly must equal hb2_evaluate_classes to
      1e-13 per pattern (relative above 1) and 1e-13 relative on lnL: this isolates the merge from the pruning;
  (B) the oracle's per-class likelihoods merged exactly must equal it at the tolerances of test_gpu_handover.py.
The per-pattern outputs siteL * 2^(-64 siteScale) are read without rounding of their own (class_merge_cases.engine_site_lnl)."""
import math

import numpy as np
import pytest

from hyphy_b200 import LikelihoodFunction, engine, synth
from oracle import port
from tests import class_merge_cases as cm

pytestmark = pytest.mark.gpu

MODES = {"fp64": engine.FLAG_FORCE_FP64, "tc": engine.FLAG_DEFAULT}    # tolerances: class_merge_cases.tolerances
RESIDENT_RTOL = {"fp64": 1e-12, "tc": 1e-9}
MERGE_TOL = 1e-13


@pytest.fixture(scope="module", autouse=True)
def _need_gpu(engine_lib):
    assert engine.device_count() > 0, "GPU tests need a CUDA device (no fallback exists)"


def tol(w, mode):
    return cm.tolerances(w, mode)


def same(a, b, rtol, atol=0.0):
    """Equal within tolerance, or the same non-finite value."""
    if not (math.isfinite(a) and math.isfinite(b)):
        return (math.isnan(a) and math.isnan(b)) or a == b
    return abs(a - b) <= max(atol, rtol * abs(b))


def sites_close(got, want, rtol, atol):
    bad = [s for s in range(len(want)) if not same(got[s], want[s], rtol, atol)]
    return bad[:5]


def hand_over(lf, P, kind=engine.MATRIX_TRANS):
    for c in range(P.shape[0]):
        lf.part.set_matrices(c, lf.all_nodes, P[c], kind)


def oracle_classes(w, P):
    out = [port.prune(w, P[c]) for c in range(P.shape[0])]
    return np.stack([o[0] for o in out]), np.stack([o[1] for o in out])


def check_merge(lf, w, P_oracle, weights, mode, label, expect=None):
    """(A) and (B) for evaluate_classes(weights) on the matrices the partition holds; returns its lnL.  expect: 'finite',
    '-inf' or 'nan' for lnL."""
    weights = np.asarray(weights, dtype=np.float64)
    rtol, atol = tol(w, mode)
    lnl, sl, ss = lf.part.evaluate_classes(weights, w.pi, want_sites=True)
    got = cm.engine_site_lnl(sl, ss)
    # (A) merge in isolation
    per = [lf.part.evaluate(c, w.pi, want_sites=True) for c in range(w.C)]
    site_a = cm.exact_site_lnl(np.stack([p[1] for p in per]), np.stack([p[2] for p in per]), weights)
    lnl_a = cm.exact_lnl(site_a, w.pattern_freq)
    bad = sites_close(got, site_a, MERGE_TOL, MERGE_TOL)
    assert not bad, f"{label}: merge of the engine's own classes, patterns {bad}: {got[bad]} vs exact {site_a[bad]}"
    assert same(lnl, lnl_a, MERGE_TOL), f"{label}: lnL {lnl!r}, exact merge of the engine's classes {lnl_a!r}"
    # (B) end to end
    osl, oss = oracle_classes(w, P_oracle)
    site_b = cm.exact_site_lnl(osl, oss, weights)
    lnl_b = cm.exact_lnl(site_b, w.pattern_freq)
    bad = sites_close(got, site_b, 0.0, atol)
    assert not bad, f"{label}: patterns {bad}: {got[bad]} vs exact oracle merge {site_b[bad]}"
    assert same(lnl, lnl_b, rtol), f"{label}: lnL {lnl!r}, exact oracle merge {lnl_b!r}"
    # per-pattern outputs: siteL finite and >= 0, 0 exactly where no class of positive weight can produce the pattern,
    # and siteL <= 1 while weights sum to at most 1 over a root vector summing to 1 (siteScale carries the rest, < 0 for L > 1).
    # siteL is NOT held above 2^-64: siteScale follows the alignment exponent of the merge (DESIGN §4.5), so a small weight
    # on the highest class (say 1e-10, without tripping the 2^-900 rescue) leaves siteL that much below it; the value
    # siteL * 2^(-64 siteScale) is what (A) and (B) pin exactly.
    ok = ~np.isnan(site_b)
    assert (sl[ok] >= 0).all() and np.isfinite(sl[ok]).all(), f"{label}: siteL out of range"
    assert ((sl[ok] == 0) == (site_b[ok] == -math.inf)).all(), f"{label}: siteL = 0 where L > 0 or the reverse"
    if weights.sum() <= 1.0 + 1e-15 and abs(w.pi.sum() - 1.0) < 1e-14:
        assert (sl[ok] <= 1.0).all(), f"{label}: siteL > 1"
    if expect == "finite":
        assert math.isfinite(lnl), f"{label}: lnL {lnl!r}"
    elif expect == "-inf":
        assert lnl == -math.inf, f"{label}: lnL {lnl!r}"
    elif expect == "nan":
        assert math.isnan(lnl), f"{label}: lnL {lnl!r}"
    return lnl, sl, ss


def gap_run(name, weights, mode, order=None, expect="finite", **kw):
    w, P = cm.gap_case(name, weights=weights, order=order, **kw)
    lf = LikelihoodFunction(w, flags=MODES[mode])
    try:
        hand_over(lf, P)
        return check_merge(lf, w, P, weights, mode, f"{name} w={list(weights)} {mode}", expect)
    finally:
        lf.close()


# ---------------------------------------------------------------------------------------------------------------------
# 1. Zero weight on the class that sits highest: the other classes are >1000 bits below it on every constant pattern

ZERO_CASES = [("d61_identity_uniform", "fp64"), ("d61_identity_uniform", "tc"), ("d20_identity_uniform", "fp64"),
              ("d4_identity_uniform", "fp64")]


@pytest.mark.parametrize("name,mode", ZERO_CASES)
def test_zero_weight_on_highest_class(name, mode):
    lnl, _, _ = gap_run(name, (0.0, 1.0), mode)
    # class 1 alone: every pattern has L = D^-leaves
    w, _ = cm.gap_case(name)
    D, L = cm.GAP_CASES[name][:2]
    want = -float(np.sum(w.pattern_freq)) * L * math.log(D)
    assert abs(lnl - want) <= tol(w, mode)[0] * abs(want), f"lnL {lnl!r}, closed form {want!r}"


@pytest.mark.parametrize("mode", ["fp64", "tc"])
@pytest.mark.parametrize("where", ["first", "middle", "last"])
def test_zero_weight_three_classes(where, mode):
    # GAP_CASES order: identity (highest), uniform, flat 1200 bits below identity
    order, weights = {"first": ((0, 1, 2), (0.0, 0.3, 0.7)), "middle": ((1, 0, 2), (0.3, 0.0, 0.7)),
                      "last": ((1, 2, 0), (0.3, 0.7, 0.0))}[where]
    gap_run("d61_three", weights, mode, order=order)


# ---------------------------------------------------------------------------------------------------------------------
# 2. Tiny weight on the highest class, with the lower class just above, just below and across the 1000-bit cutoff

@pytest.mark.parametrize("mode", ["fp64", "tc"])
@pytest.mark.parametrize("name,weights", [("d61_gap1010", (1e-305, 1.0)), ("d61_gap990", (1e-305, 1.0)),
                                          ("d61_gap1030", (1e-305, 1.0)), ("d61_gap1062", (5e-320, 1.0))])
def test_tiny_weight_on_highest_class(name, weights, mode):
    gap_run(name, weights, mode)


# ---------------------------------------------------------------------------------------------------------------------
# 3. Classes far apart with ordinary weights: the dominant class wins; L > 1 with unnormalised weights or a root of ones

@pytest.mark.parametrize("mode", ["fp64", "tc"])
@pytest.mark.parametrize("name", ["d61_gap500", "d61_gap1100", "d61_gap3000"])
def test_far_apart_ordinary_weights(name, mode):
    _, sl, ss = gap_run(name, (0.4, 0.6), mode)
    w, _ = cm.gap_case(name)
    const = cm.is_constant(w)
    # the identity class dominates by >= 495 bits: every constant pattern is log(0.4 / D), exactly
    got = cm.engine_site_lnl(sl, ss)[const]
    assert np.abs(got - math.log(0.4 / 61)).max() <= tol(w, mode)[1]


@pytest.mark.parametrize("mode", ["fp64", "tc"])
def test_likelihood_above_one(mode):
    _, sl, ss = gap_run("d61_above", (3.0, 4.0), mode)
    assert (ss < 0).all() and (sl <= 1.0).all() and (sl > 0).all()
    _, sl, ss = gap_run("d61_gap500", (0.4, 0.6), mode, pi=np.ones(61))
    assert (sl > 0).all()


# ---------------------------------------------------------------------------------------------------------------------
# 4. Impossible classes: an identity class cannot produce a pattern whose leaves differ

@pytest.mark.parametrize("mode", ["fp64", "tc"])
def test_impossible_patterns(mode):
    name = "d61_identity_uniform"
    gap_run(name, (0.5, 0.5), mode, n_free=6)                         # the uniform class carries them: finite
    gap_run(name, (1.0, 0.0), mode, n_free=6, expect="-inf")          # nothing of positive weight can: -inf
    S = 300
    zero = tuple(range(S - 6, S))
    _, sl, _ = gap_run(name, (1.0, 0.0), mode, n_free=6, zero_freq=zero)   # ... unless those patterns have frequency 0
    assert (sl[S - 6:] == 0).all() and (sl[:S - 6] > 0).all()


# ---------------------------------------------------------------------------------------------------------------------
# 5. NaN

@pytest.mark.parametrize("mode", ["fp64", "tc"])
def test_nan(mode):
    name = "d61_three"
    w, P = cm.gap_case(name)
    Pn = P.copy()
    Pn[1, 3] = np.nan                                                 # class 1 (uniform), one branch
    lf = LikelihoodFunction(w, flags=MODES[mode])
    try:
        hand_over(lf, Pn)
        label = f"nan {mode}"
        check_merge(lf, w, Pn, (0.2, 0.3, 0.5), mode, label, expect="nan")
        lnl, sl, ss = check_merge(lf, w, Pn, (0.2, 0.0, 0.5), mode, label, expect="finite")
        # a NaN class of weight 0 is not there at all: the same as the merge of the other two
        site = cm.exact_site_lnl(np.stack([port.prune(w, P[c])[0] for c in (0, 2)]),
                                 np.stack([port.prune(w, P[c])[1] for c in (0, 2)]), (0.2, 0.5))
        assert same(lnl, cm.exact_lnl(site, w.pattern_freq), tol(w, mode)[0])
        assert math.isnan(lf.part.evaluate_classes(np.array([0.2, np.nan, 0.5]), w.pi))
        hand_over(lf, P)
        assert math.isnan(lf.part.evaluate_classes(np.array([np.nan, 0.3, 0.7]), w.pi))
        check_merge(lf, w, P, (0.0, 0.3, 0.7), mode, label, expect="finite")
    finally:
        lf.close()


# ---------------------------------------------------------------------------------------------------------------------
# 6. Recovery after -inf: the flag and the ticket counter of the root reduction are re-armed

def _generic(D, C, n_taxa=12, S=300, seed=20261016):
    """A simulated alignment of S sites (duplicate columns kept as patterns of frequency 1) with C rate classes."""
    w = synth.generic_workload(D, n_taxa, S, C, seed=seed, mean_t=0.1)
    w.leaf_states = np.ascontiguousarray(w.leaf_states[:, w.site_to_pattern])
    w.pattern_freq = np.ones(S, dtype=np.int64)
    w.site_to_pattern = np.arange(S, dtype=np.int64)
    return w


@pytest.mark.parametrize("D,mode", [(20, "fp64"), (61, "fp64"), (61, "tc")])
def test_recovery_after_minus_inf(D, mode):
    w = _generic(D, 2)
    wts = np.array([0.4, 0.6])
    Qt = w.Qt()
    ident = np.broadcast_to(np.eye(D), (2,) + Qt.shape[1:]).copy()
    b = 3
    fresh = LikelihoodFunction(w, flags=MODES[mode])
    lf = LikelihoodFunction(w, flags=MODES[mode])
    try:
        hand_over(fresh, Qt, engine.MATRIX_RATE)
        want = {"evaluate": fresh.part.evaluate(1, w.pi), "classes": fresh.part.evaluate_classes(wts, w.pi)}
        fresh.part.branch_cache_build(b, w.pi)
        for c in range(2):
            fresh.part.set_matrices(c, [b], Qt[c, b][None] * 1.7)
        want["branch_cache"] = fresh.part.branch_cache_evaluate(wts)
        hand_over(fresh, Qt, engine.MATRIX_RATE)
        want["resident"] = fresh.part.time_resident(wts, w.pi, iters=1)[2]

        def poison():
            hand_over(lf, ident)                                      # identity matrices: every variable pattern is impossible
            assert lf.part.evaluate_classes(wts, w.pi) == -math.inf
            hand_over(lf, Qt, engine.MATRIX_RATE)

        poison()
        assert lf.part.evaluate(1, w.pi) == want["evaluate"]
        poison()
        assert lf.part.evaluate_classes(wts, w.pi) == want["classes"]
        poison()
        lf.part.evaluate_classes(wts, w.pi)
        lf.part.branch_cache_build(b, w.pi)
        for c in range(2):
            lf.part.set_matrices(c, [b], Qt[c, b][None] * 1.7)
        assert lf.part.branch_cache_evaluate(wts) == want["branch_cache"]
        poison()
        assert lf.part.time_resident(wts, w.pi, iters=1)[2] == want["resident"]
    finally:
        lf.close()
        fresh.close()


# ---------------------------------------------------------------------------------------------------------------------
# 7. Many classes on every kernel family, with a weight of 0 and a weight of 1e-200 among them

@pytest.mark.parametrize("C", [8, 16])
@pytest.mark.parametrize("D,mode", [(4, "fp64"), (20, "fp64"), (61, "fp64"), (61, "tc")])
def test_many_classes(D, mode, C):
    w = _generic(D, C, seed=20261016 + C)
    rng = np.random.default_rng(C + D)
    wts = rng.dirichlet(np.ones(C))
    wts[1], wts[C - 2] = 0.0, 1e-200
    Qt = w.Qt()
    P = np.stack([np.stack([port.expm(Qt[c, b]) for b in range(Qt.shape[1])]) for c in range(C)])
    rtol, _ = tol(w, mode)
    lf = LikelihoodFunction(w, flags=MODES[mode])
    try:
        hand_over(lf, Qt, engine.MATRIX_RATE)
        full, _, _ = check_merge(lf, w, P, wts, mode, f"D={D} C={C} {mode}", expect="finite")
        # the replay behind bench.py's value
        res = lf.part.time_resident(wts, w.pi, iters=1)[2]
        assert same(res, full, RESIDENT_RTOL[mode]), f"resident {res!r}, compute {full!r}"
        # partial update of one branch in every class, then the full evaluation of the same matrices
        b = 5
        Q2 = Qt.copy()
        Q2[:, b] *= 1.4
        for c in range(C):
            lf.part.set_matrices(c, [b], Q2[c, b][None])
        part_l = lf.part.evaluate_classes(wts, w.pi, update_nodes=[b])
        full2 = lf.part.evaluate_classes(wts, w.pi)
        if mode == "fp64":
            assert part_l == full2, f"partial {part_l!r}, full {full2!r}"
        else:
            assert same(part_l, full2, 1e-12)
        P2 = P.copy()
        P2[:, b] = np.stack([port.expm(Q2[c, b]) for c in range(C)])
        check_merge(lf, w, P2, wts, mode, f"D={D} C={C} {mode} after partial update", expect="finite")
        # branch-cache probe with the weights: only branch b changes again
        lf.part.evaluate_classes(wts, w.pi)
        lf.part.branch_cache_build(b, w.pi)
        for c in range(C):
            lf.part.set_matrices(c, [b], Qt[c, b][None])
        probe = lf.part.branch_cache_evaluate(wts)
        back = lf.part.evaluate_classes(wts, w.pi)
        assert same(probe, back, max(rtol, 1e-12)), f"probe {probe!r}, full {back!r}"
        assert same(back, full, 0.0 if mode == "fp64" else 1e-12), f"back {back!r}, first {full!r}"
    finally:
        lf.close()
