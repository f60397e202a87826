"""CPU suite: the exact rate-class merge of tests/class_merge_cases.py against the oracle with ordinary weights and
against hand-computed sums at the edges, and the scale gaps of the workloads tests/test_gpu_class_merge.py relies on."""
import math

import numpy as np
import pytest

from oracle import port
from tests import class_merge_cases as cm
from tests import golden_cases as gc


def per_class(w, P):
    out = [port.prune(w, P[c]) for c in range(P.shape[0])]
    return np.stack([o[0] for o in out]), np.stack([o[1] for o in out])


@pytest.mark.parametrize("name", ["mg94_8x60_c4_ambig", "c1_hky85_8x500"])
def test_exact_merge_matches_oracle_with_ordinary_weights(name):
    w, _ = gc.load(name)
    Qt = w.Qt()
    P = np.stack([np.stack([port.expm(Qt[c, b], w.D > 20) for b in range(Qt.shape[1])]) for c in range(w.C)])
    sl, ss = per_class(w, P)
    site = cm.exact_site_lnl(sl, ss, w.class_weights)
    ref, ref_site = port.lnl(w)
    got = cm.exact_lnl(site, w.pattern_freq)
    assert abs(got - ref) <= 1e-13 * abs(ref), f"{got!r} vs oracle {ref!r}"
    assert np.abs(site - ref_site).max() <= 1e-12


@pytest.mark.parametrize("name", list(cm.GAP_CASES))
def test_gap_cases_sit_where_they_say(name):
    lo, hi = cm.GAP_CASES[name][3]
    w, P = cm.gap_case(name, S=24, n_free=4)
    sl, ss = per_class(w, P)
    e = cm.class_exponents(sl, ss)
    const = cm.is_constant(w)
    gap = e[0, const] - e[1, const]
    assert lo < gap.min() and gap.max() < hi, f"gap {gap.min():.1f}..{gap.max():.1f} bits, expected ({lo}, {hi})"
    # an identity class cannot produce a pattern whose leaves differ; every other class can
    assert const.sum() == w.S - 4 and (sl[0, ~const] == 0).all() and (sl[1:, ~const] > 0).all()
    # the flat classes follow their closed form (log2, to rounding of the products)
    D, _, specs, _ = cm.GAP_CASES[name]
    for c, sp in enumerate(specs):
        if sp != "identity":
            assert np.abs(e[c] - cm.flat_log2(w.tree, D, cm.flat_entry(sp, w.tree, D))).max() < 1e-6


def test_exact_merge_by_hand():
    # class 0 at 2^-2000 (too small for a double), class 1 at 2^-3000, class 2 at 0.5
    sl = np.array([[0.5, 0.5, 0.75], [0.25, 0.5, 0.0], [0.5, 0.0, 0.0]])
    ss = np.array([[31, 0, 0], [47, 0, 0], [0, 0, 0]])
    ln2 = math.log(2.0)
    # ordinary weights: the big class wins, the others still count (exactly)
    got = cm.exact_site_lnl(sl, ss, [0.25, 0.25, 0.5])
    assert got[0] == pytest.approx(math.log(0.25), rel=1e-15)
    assert got[1] == pytest.approx(math.log(0.25 * 0.5 + 0.25 * 0.5), rel=1e-15)
    assert got[2] == pytest.approx(math.log(0.25 * 0.75), rel=1e-15)
    # zero weight on the big class: the pattern is the tiny classes', far below any double
    got = cm.exact_site_lnl(sl, ss, [1.0, 2.0, 0.0])
    assert got[0] == pytest.approx(math.log(0.5) - 64 * 31 * ln2, abs=1e-12)
    assert got[2] == pytest.approx(math.log(0.75), rel=1e-15)
    # every class of weight 0 (or with weight 0 except classes at 0): -inf
    assert cm.exact_site_lnl(sl, ss, [0.0, 0.0, 0.0]).tolist() == [-math.inf] * 3
    assert cm.exact_site_lnl(sl, ss, [0.0, 1.0, 1.0])[2] == -math.inf


def test_exact_merge_nan_and_weights():
    sl = np.array([[0.5, np.nan], [0.25, 0.5]])
    ss = np.zeros((2, 2), dtype=np.int64)
    # NaN in a class of weight 0 is ignored; with weight > 0 it is NaN; a NaN weight is NaN
    got = cm.exact_site_lnl(sl, ss, [1.0, 1.0])
    assert got[0] == pytest.approx(math.log(0.75), rel=1e-15) and math.isnan(got[1])
    got = cm.exact_site_lnl(sl, ss, [0.0, 1.0])
    assert got == pytest.approx([math.log(0.25), math.log(0.5)], rel=1e-15)
    assert np.isnan(cm.exact_site_lnl(sl, ss, [np.nan, 1.0])).all()
    # unnormalised weights (sum 7): L > 1
    got = cm.exact_site_lnl(np.array([[1.0], [1.0]]), np.array([[0], [-1]]), [3.0, 4.0])
    assert got[0] == pytest.approx(math.log(3.0 + 4.0 * 2.0 ** 64), rel=1e-15)
    # a subnormal weight keeps every bit: 5e-320 * 2^1000 * 0.5
    got = cm.exact_site_lnl(np.array([[0.5]]), np.array([[-15]]), [5e-320])
    want = math.log(5e-320 / 2 ** -1074) - 1074 * math.log(2.0) + 960 * math.log(2.0) + math.log(0.5)
    assert got[0] == pytest.approx(want, abs=1e-12)


def test_exact_lnl_frequencies():
    site = np.array([-1.0, -math.inf, -2.5, np.nan])
    assert cm.exact_lnl(site, [2, 0, 1, 0]) == -4.5
    assert cm.exact_lnl(site, [2, 1, 1, 0]) == -math.inf
    assert math.isnan(cm.exact_lnl(site, [2, 0, 1, 1]))


def test_exact_log_far_from_one():
    """Against 60-digit decimal logs, for sums shaped like the gap cases: numerator and denominator of thousands of bits
    whose ratio is near 1, and plain ratios far from it."""
    from decimal import Decimal, getcontext
    from fractions import Fraction
    getcontext().prec = 60
    two = Fraction(2)
    cases = [r * two ** k for k in (-3000, -1100, -64, 0, 700, 3000)
             for r in (Fraction(1, 3), Fraction(5, 7), Fraction(3, 2))]
    for gap in (500, 1100, 3000):
        # 0.4 * 2^-6 + 0.6 * 2^(-6-gap) * (odd mantissa): a near-1 ratio of two integers of about `gap` bits
        cases.append(Fraction(0.4) / 64 + Fraction(0.6) * Fraction(3 ** 40 + 1, 3 ** 40) * two ** (-6 - gap))
        cases.append((Fraction(3 ** 700 + 1, 3 ** 700)) * two ** -gap)
        cases.append(1 + two ** -gap)
    for x in cases:
        want = Decimal(x.numerator).ln() - Decimal(x.denominator).ln()
        got = cm.exact_log(x)
        assert abs(Decimal(got) - want) <= Decimal(math.ulp(float(want))), (float(x) if x > 2 ** -1000 else "tiny", got, want)
