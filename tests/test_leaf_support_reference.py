"""CPU suite: tests/leaf_support_reference.py, the reference of tests/test_gpu_leaf_support.py, and the reference binary's
leaf imputation fixtures.

The outside-pass restatement equals the reference's own procedure (every leaf forced to every state, normalised); rows
sum to 1 and do not depend on their own leaf's code; the fixtures are the workloads the GPU file builds and hold
probabilities; and -- what makes the GPU tests able to see a kernel bug at all -- each plausible bug of MUTATIONS moves
an entry of the GPU file's own workloads by more than ten times the tolerance that file holds the engine to."""
import math
import os

import numpy as np
import pytest

from tests import batch_reference as br
from tests import golden_cases as gc
from tests import leaf_support_reference as lsr
from tests import test_gpu_leaf_support as G

BIG = 1e-6                          # entries compared relatively


def _args(case, s, expm, col=None):
    return (case.w.tree, expm, case.V[s], case.W[s] if case.mix else None, case.branch_k,
            case.w.leaf_states[:, case.pats[s]] if col is None else col, case.w.ambig, case.root)


def _close(a, b, rel, abs_):
    a, b = np.asarray(a, dtype=br.LD), np.asarray(b, dtype=br.LD)
    err = np.abs(a - b)
    big = np.abs(b) >= BIG
    return float(err.max()) <= abs_ and float((err[big] / np.abs(b[big])).max()) <= rel


CASES = [(33, False, True), (48, True, False), (64, False, False), (61, True, True)]


@pytest.mark.parametrize("D,reversible,mix", CASES, ids=[f"{d}{'' if r else '-nonrev'}{'-mix' if m else '-plain'}"
                                                         for d, r, m in CASES])
def test_outside_equals_brute_force(D, reversible, mix):
    case, expm = G.sweep_support_case(D, reversible, mix)
    for s in range(3):
        a = lsr.brute_support(*_args(case, s, expm))
        b = lsr.outside_support(*_args(case, s, expm))
        assert np.all(np.isfinite(a))
        assert _close(b, a, 1e-15, 1e-18), s
        assert np.abs(a.sum(axis=1) - 1).max() <= 1e-17


def test_outside_equals_brute_force_on_a_wide_tree():
    """poly7 at 48 states: leaves under the root and under a seven-child node."""
    case, expm = G.shape_support_case("poly7", True)
    a = lsr.brute_support(*_args(case, 0, expm))
    assert _close(lsr.outside_support(*_args(case, 0, expm)), a, 1e-15, 1e-18)


def test_row_ignores_own_code():
    """Leaf l's row is the same, bit for bit in long double, whatever l's own code: every state and ambiguity row."""
    case, expm = G.sweep_support_case(48, False, True)
    col = case.w.leaf_states[:, case.pats[0]].copy()
    base = lsr.outside_support(*_args(case, 0, expm, col))
    brute = lsr.brute_support(*_args(case, 0, expm, col))
    for l in (0, 4, case.w.tree.n_leaves - 1):
        for code in [0, 7, case.w.D - 1] + [-(r + 1) for r in range(len(case.w.ambig))]:
            c2 = col.copy()
            c2[l] = code
            assert np.array_equal(lsr.outside_support(*_args(case, 0, expm, c2))[l], base[l]), (l, code)
            assert _close(lsr.brute_support(*_args(case, 0, expm, c2))[l], brute[l], 1e-16, 1e-19), (l, code)


def test_zero_root_gives_nan_rows():
    case, expm = G.sweep_support_case(33, False, False)
    args = list(_args(case, 0, expm))
    args[-1] = np.zeros(case.w.D)
    assert np.all(np.isnan(lsr.outside_support(*args))) and np.all(np.isnan(lsr.brute_support(*args)))


@pytest.mark.parametrize("name", list(G.FIXTURES))
def test_fixture_is_consistent(name):
    """The fixture is the workload the GPU file builds; its rows are probabilities; sites of one pattern share a row;
    its lnL is the case's."""
    w, g0 = gc.load(name)
    g = np.load(os.path.join(gc.GOLDEN_DIR, name + "_impute.npz"))
    assert str(g["checksum"]) == gc.checksum(w)
    assert float(g["lnL"]) == g0["lnL"]
    sup = g["support"]
    assert sup.shape == (len(w.site_to_pattern), w.tree.n_leaves, w.D)
    assert np.all(sup >= 0) and np.abs(sup.sum(axis=2) - 1).max() <= 1e-12
    for p in range(w.S):
        sites = np.nonzero(w.site_to_pattern == p)[0]
        assert np.all(sup[sites] == sup[sites[:1]]), p
    assert np.abs(sup - sup[:, :, :1]).max() > 0.1                          # not uniform


@pytest.mark.parametrize("name", list(G.FIXTURES))
def test_fixture_matches_long_double_reference(name):
    """A few patterns of the fixture against the long-double outside pass: the reference binary's rows are the
    predictive distributions this file restates."""
    w, _ = gc.load(name)
    g = np.load(os.path.join(gc.GOLDEN_DIR, name + "_impute.npz"))
    V, W, branch_k = G.fixture_sets(w)
    ex = G.CodonExpm(w, True)
    first = np.array([np.nonzero(w.site_to_pattern == p)[0][0] for p in range(w.S)])
    for p in (0, w.S // 2, w.S - 1):
        ref = lsr.outside_support(w.tree, ex, V, W, branch_k, w.leaf_states[:, p], w.ambig, w.pi).astype(np.float64)
        assert np.abs(g["support"][first[p]] - ref).max() <= 1e-9, p


# ---------------------------------------------------------------------------------------------------------------------
# mutations: each plausible kernel bug moves an entry of a GPU file's workload beyond that file's tolerance
# ---------------------------------------------------------------------------------------------------------------------
def _sweep(D, reversible, mix):
    def case():
        c, ex = G.sweep_support_case(D, reversible, mix)
        return _args(c, 0, ex)
    return case


def _shape(shape):
    def case():
        c, ex = G.shape_support_case(shape, True)
        return _args(c, 0, ex)
    return case


MUTATION_CASES = {                  # mutation: a workload of tests/test_gpu_leaf_support.py
    "posterior": _sweep(48, False, False),
    "leaf_through_P": _sweep(48, False, True),
    "leaf_component0": _sweep(33, False, True),
    "outside_no_siblings": _sweep(61, True, False),
    "sibling_self": _sweep(64, False, True),
    "root_ones": _sweep(48, True, True),
    "drop_third_child": _shape("poly7"),
}


def test_every_mutation_has_a_case():
    assert set(MUTATION_CASES) == set(lsr.MUTATIONS)


@pytest.mark.parametrize("mutation", list(MUTATION_CASES))
def test_mutation_moves_an_entry_beyond_tolerance(mutation):
    args = MUTATION_CASES[mutation]()
    ref = lsr.outside_support(*args).astype(np.float64)
    assert np.array_equal(ref, lsr.outside_support(*args, mutate=()).astype(np.float64))
    mut = lsr.outside_support(*args, mutate=(mutation,)).astype(np.float64)
    big = ref >= BIG
    with np.errstate(invalid="ignore"):
        err = np.abs(mut[big] - ref[big]) / ref[big]
    shift = float(np.where(np.isnan(err), np.inf, err).max())
    print(f"{mutation}: largest relative shift {shift:.2e} against tolerance {G.TOL_REL:.0e}")
    assert shift > 10 * G.TOL_REL or math.isinf(shift), (mutation, shift)
