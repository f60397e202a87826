"""CPU suite: the reference builders of tests/handover_cases.py, which the GPU hand-over tests (tests/test_gpu_handover.py)
compare the engine with.  `assemble` must reproduce the workloads' own dense matrices from their compiled form, the new
templates must describe reversible rate matrices, and the oracle's expm must agree with scipy on them."""
import numpy as np
import pytest
import scipy.linalg

from hyphy_b200 import synth
from oracle import port
from tests import handover_cases as hc


@pytest.mark.parametrize("w", [synth.codon_workload(8, 30, 4), synth.codon_workload(8, 30, 1), synth.nucleotide_workload(8, 50)],
                         ids=lambda w: w.name)
def test_assemble_reproduces_the_workloads_dense_matrices(w):
    ei, ef, _, cf = w.compiled_template()
    V, Qt = w.compiled_values(), w.Qt()
    for c in range(w.C):
        for b in range(w.tree.n_branches):
            np.testing.assert_allclose(hc.assemble(ei, ef, V[c, b], cf, w.D), Qt[c, b], rtol=0, atol=1e-15)


def test_assemble_multiplies_columns_and_sets_the_diagonal():
    Q = hc.assemble([1, 2, 3], [0, 1, 0], [2.0, 3.0], [0.5, 0.25], 2)     # index 3 = (1, 1): a diagonal entry is ignored
    np.testing.assert_array_equal(Q, [[-2.0 * 0.25, 2.0 * 0.25], [3.0 * 0.5, -3.0 * 0.5]])


def _templates():
    g = hc.gy94_template()
    yield "gy94", g, g.Q(hc.gy94_rates(2.5, 0.4) * 0.3)
    g2 = g.with_freqs(hc.codon_pi(3))
    yield "gy94-other-pi", g2, g2.Q(hc.gy94_rates(4.0, 1.7) * 0.05)
    for D in (20, 48):
        t, x = hc.gtr_template(D, D)
        yield f"gtr{D}", t, t.Q(x * 0.2)


@pytest.mark.parametrize("name,t,Q", list(_templates()), ids=[n for n, _, _ in _templates()])
def test_templates_are_reversible_rate_matrices(name, t, Q):
    assert Q.shape == (t.D, t.D) and len(set(t.ei.tolist())) == len(t.ei)
    assert np.abs(Q.sum(axis=1)).max() <= 1e-15 * np.abs(Q).max() * t.D
    off = ~np.eye(t.D, dtype=bool)
    assert np.all(Q[off] >= 0) and np.all(np.diag(Q) < 0)
    F = t.cf[:, None] * Q
    np.testing.assert_allclose(F, F.T, rtol=1e-14, atol=0)
    assert abs(t.cf.sum() - 1.0) < 1e-14 and np.all(t.cf > 0)


@pytest.mark.parametrize("name,t,Q", list(_templates()), ids=[n for n, _, _ in _templates()])
@pytest.mark.parametrize("scale", [1e-6, 0.1, 1.0, 2.29 / 2, 2.31 / 2, 8.0])
def test_oracle_expm_matches_scipy_on_templates(name, t, Q, scale):
    A = Q * (scale / hc.inf_norm(Q) * 2.0 if scale > 0.5 else scale)
    np.testing.assert_allclose(port.expm(A), scipy.linalg.expm(A), rtol=0, atol=1e-13)


def test_gtr_template_has_unit_mean_rate():
    for D in (20, 48):
        t, x = hc.gtr_template(D, D)
        assert abs(-(t.cf * np.diag(t.Q(x))).sum() - 1.0) < 1e-13


def test_oracle_lnl_over_classes_matches_port_lnl():
    """oracle_lnl (per-class pruning, mixed over classes) agrees with the oracle's own class mixture."""
    w = synth.codon_workload(10, 40, 4)
    Qt = w.Qt()
    P = np.stack([[port.expm(q) for q in Qt[c]] for c in range(w.C)])
    ref, site = port.lnl(w, Qt, sparse_storage=False)
    got, gsite = hc.oracle_lnl(w, P)
    assert abs(got - ref) <= 1e-12 * abs(ref)
    np.testing.assert_allclose(gsite, site, rtol=0, atol=1e-11)
