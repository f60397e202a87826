"""CPU suite for tests/resident_reference.py, the reference of the resident evaluation path: it agrees with scipy's
exponential, with the oracle's fp64 pruning, pinned nodes and conditionals, and with batch_reference.prune_ld; every
restated kernel bug moves the GPU file's workloads beyond ten times their tolerances; and the classification by shares
of the weight passes the oracle suites' bounds, which is why they could not see it."""
import numpy as np
import pytest
import scipy.linalg

from oracle import port
from tests import batch_reference as br
from tests import resident_reference as rr
from tests.test_gpu_resident_reference import (LENGTHS, SHARE_MOVES, SWEEP_TREE, TOL, Case, family, near_proportional, probe_pattern,
                                               rel, switch_lengths)

OLD_SITE_ATOL, OLD_LNL_RTOL = 1e-8, 1e-10          # test_gpu_shapes.MODES["fp64"]


def oracle_sites(w, P):
    sl, ss = port.prune(w, np.asarray(P, dtype=np.float64))
    return np.log(sl) - 64.0 * np.log(2.0) * ss


@pytest.mark.parametrize("D", [2, 5, 20, 32, 48, 64])
def test_expm_matches_scipy(D):
    """Every switch-point length of the GPU file: long double against scipy's Pade expm to its own accuracy."""
    case = Case(SWEEP_TREE, D, rates=[1.0], weights=[1.0], S=40, seed=2)
    Q = br.dense(case.t, case.t.base)
    for kind in (["small"] if D <= 32 else ["dmma", "poly"]):
        for label, x in switch_lengths(Q, kind):
            got = np.asarray(case.expm(Q * x), dtype=np.float64)
            ref = scipy.linalg.expm(Q * x)
            assert np.abs(got - ref).max() <= (1e-11 if label == "saturating" else 1e-13), (kind, label)


@pytest.mark.parametrize("D,reversible", [(4, True), (20, True), (48, True), (61, True), (4, False), (48, False)])
def test_reference_agrees_with_oracle(D, reversible):
    """Per-class log-likelihoods, a pinned internal node and the conditionals against the oracle's fp64 recursion on the
    same (oracle-exponentiated) matrices; the class merge against a direct long-double sum."""
    case = Case(SWEEP_TREE, D, reversible, S=80, seed=1)
    w = case.w
    L, I = w.tree.n_leaves, w.tree.n_internal
    per = []
    for c in range(len(case.rates)):
        P = np.stack([port.expm(A, False) for A in case.dense(c)])
        got, cond = rr.class_sites(w.tree, P, case.cols(), w.ambig, case.root, want_cond=True)
        assert float(rel(got, oracle_sites(w, P)).max()) <= 1e-13
        fs = np.random.default_rng(c).integers(0, D, w.S)
        pinned = rr.class_sites(w.tree, P, case.cols(), w.ambig, case.root, pin=(L + I // 2, fs))
        sl, ss = port.prune_forced(w, P, L + I // 2, fs)
        assert float(rel(pinned, np.log(sl) - 64.0 * np.log(2.0) * ss).max()) <= 1e-13
        _, _, ocond = port.prune(w, P, want_cond=True)
        for i in range(I):
            o = ocond[i] / ocond[i].max(axis=1, keepdims=True)
            assert np.abs(np.asarray(cond[i], dtype=np.float64) - o).max() <= 1e-13
        per.append(got)
    merged = rr.merge(per, w.class_weights)
    direct = np.log(sum(rr.LD(wc) * np.exp(p) for wc, p in zip(w.class_weights, per) if wc > 0))
    assert float(rel(merged, direct).max()) <= 1e-17


def test_prune_ld_is_the_same_recursion():
    case = Case(SWEEP_TREE, 48, S=60, seed=1)
    P = case.P()[2]
    a = br.prune_ld(case.tree, P, case.cols(), case.w.ambig, case.root)
    assert np.array_equal(a, rr.class_sites(case.tree, P, case.cols(), case.w.ambig, case.root))


def test_zero_weight_class_never_enters():
    """A zero-weight class whose likelihood is 0 (log -inf) or NaN leaves the merge untouched."""
    per = np.array([[-3.0, -4.0], [-np.inf, np.nan], [-2.5, -7.0]], dtype=rr.LD)
    w = np.array([0.4, 0.0, 0.6])
    ref = np.log(0.4 * np.exp(per[0]) + 0.6 * np.exp(per[2]))
    assert float(np.abs(rr.merge(per, w) - ref).max()) <= 1e-18


# ---------------------------------------------------------------------------------------------------------------------
# mutations
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mutation", ["fp32_root", "fp32_class_weights"])
@pytest.mark.parametrize("D,mode", [(4, "fp64"), (20, "fp64"), (48, "fp64"), (64, "fp64")])
def test_staging_mutations_are_caught(mutation, D, mode):
    """The sweep workloads of the GPU file: one pattern moves by more than ten times its family's per-pattern bound."""
    case = Case(SWEEP_TREE, D, S=200, seed=1)
    clean, _ = rr.evaluate(case.tree, case.P(), case.cols(), case.w.ambig, case.root, case.w.class_weights)
    bad, _ = rr.evaluate(case.tree, case.P(), case.cols(), case.w.ambig, case.root, case.w.class_weights, {mutation})
    assert float(rel(bad, clean).max()) > 10 * TOL[family(D, mode)]["site"]


def near_proportional_probe(D, handover, move, mutate):
    """The near-proportional case of the GPU file (in-batch route): branch 1's matrix and its probe pattern, exponentiated
    as the shared-powers stage would under `mutate`.  Returns (clean P[leaf], P[leaf], clean sites, sites, case)."""
    case = Case(SWEEP_TREE, D, rates=[1.0], weights=[1.0], S=100, seed=3)
    compiled = handover == "compiled"
    leaf = 1
    case.tree.t[leaf] = LENGTHS[-1]
    A0, V0 = case.dense(0), case.values(0)
    v, f = near_proportional(A0[leaf], V0[leaf] if compiled else A0[leaf].ravel(), move, compiled)
    A = br.dense(case.t, v) if compiled else v.reshape(D, D)
    if compiled:
        i, j = divmod(int(case.t.ei[np.nonzero(case.t.ef == f)[0][0]]), D)
    else:
        i, j = divmod(int(f), D)
    case.w.leaf_states[:, 0] = probe_pattern(case, leaf, i, j)
    sub = rr.substitute(A, A0[0], v if compiled else None, V0[0] if compiled else None, mutate)
    P = case.P()[0].copy()
    Pm = P.copy()
    P[leaf], Pm[leaf] = case.expm(A), case.expm(sub)
    clean = rr.class_sites(case.tree, P, case.cols(), case.w.ambig, case.root)
    bad = rr.class_sites(case.tree, Pm, case.cols(), case.w.ambig, case.root)
    return P[leaf], Pm[leaf], clean, bad, case


@pytest.mark.parametrize("handover", ["dense", "compiled"])
@pytest.mark.parametrize("D", [48, 61, 64])
def test_share_rule_flags_what_the_value_rule_refuses(D, handover):
    """Moves up to 1e-13 of a share pass the share rule, larger ones do not; the value rule refuses every move and still
    accepts exact scalings (Q t from the host, formula values times t)."""
    case = Case(SWEEP_TREE, D, rates=[1.0], weights=[1.0], S=40, seed=3)
    compiled = handover == "compiled"
    A0, V0 = case.dense(0), case.values(0)
    ref = V0[0] if compiled else A0[0]
    for move in SHARE_MOVES:
        v, _ = near_proportional(A0[1], V0[1] if compiled else A0[1].ravel(), move, compiled)
        assert rr.share_flagged(v, ref) == (move < 1e-13), move
        assert not rr.value_flagged(v, ref), move
    Q = br.dense(case.t, case.t.base)
    for b in range(case.tree.n_branches):
        assert rr.value_flagged(V0[b] if compiled else A0[b], ref)
        assert rr.value_flagged(Q * case.tree.t[b], Q * case.tree.t[0])


@pytest.mark.parametrize("handover", ["dense", "compiled"])
@pytest.mark.parametrize("D", [48, 61, 64])
def test_share_proportionality_is_caught_and_passed_the_old_bounds(D, handover):
    """At share moves of 0.5e-13 and 0.9e-13 the probe's matrix and its pattern move by more than ten times the lanes
    family's bounds, yet the whole workload stays inside the oracle suites' fp64 bounds (1e-8 per pattern, 1e-10 of
    lnL)."""
    for move in (0.5e-13, 0.9e-13):
        Pc, Pm, clean, bad, case = near_proportional_probe(D, handover, move, {"share_proportionality"})
        assert float(np.abs(Pm - Pc).max()) > 10 * TOL["lanes"]["matrix"]
        assert float(rel(bad, clean).max()) > 10 * TOL["lanes"]["site"]
        assert float(np.abs(bad - clean).max()) <= OLD_SITE_ATOL
        f = case.w.pattern_freq
        assert float(rel((f * bad).sum(), (f * clean).sum())) <= OLD_LNL_RTOL
    # above the share bound nothing is substituted
    Pc, Pm, clean, bad, _ = near_proportional_probe(D, handover, 1.1e-13, {"share_proportionality"})
    assert np.array_equal(Pc, Pm) and np.array_equal(clean, bad)
