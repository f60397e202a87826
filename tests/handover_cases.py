"""Reference builders for the hand-over tests: the dense rate matrix a compiled hand-over describes, templates with column
frequencies (61-state GY94 shape, GTR shape for any state count) and oracle transition matrices and likelihoods for a
tree whose branches carry matrices of several templates, mixtures or dense inputs.  No test functions live here."""
import dataclasses

import numpy as np

from hyphy_b200 import synth
from oracle import port

EXPM_POLY_THETA = 2.3        # hb2_kernels_fp64.cuh: the shared-powers polynomial needs no squaring up to this norm


def assemble(ei, ef, values, col_freq, D):
    """The dense Q a compiled hand-over describes (load_rate_matrix in hb2_kernels_fp64.cuh): entry ei[e] = row * D + col
    holds values[ef[e]] * col_freq[col]; the diagonal is minus the off-diagonal row sum."""
    r, c = np.divmod(np.asarray(ei, dtype=np.int64), D)
    v = np.asarray(values, dtype=np.float64)[np.asarray(ef, dtype=np.int64)]
    if col_freq is not None:
        v = v * np.asarray(col_freq, dtype=np.float64)[c]
    off = r != c
    Q = np.zeros((D, D))
    Q[r[off], c[off]] = v[off]
    Q[np.diag_indices(D)] = -Q.sum(axis=1)
    return Q


@dataclasses.dataclass
class Template:
    """A compiled template: entry index and formula of every off-diagonal entry, number of formulas, column frequencies."""
    ei: np.ndarray
    ef: np.ndarray
    nF: int
    cf: np.ndarray | None
    D: int

    def Q(self, values, cf="current"):
        return assemble(self.ei, self.ef, values, self.cf if isinstance(cf, str) else cf, self.D)

    def define(self, part, tid):
        part.set_rate_template_id(tid, self.ei, self.ef, self.nF, self.cf)

    def with_freqs(self, cf):
        return dataclasses.replace(self, cf=None if cf is None else np.asarray(cf, dtype=np.float64))


def gy94_template(col_freq=None):
    """61 codon states, GY94 shape: one formula per (transition or transversion, synonymous or not) -- formula
    2 * transition + nonsynonymous -- and the codon frequencies as column multipliers (default: the CF3x4 codon pi)."""
    ei, ef = [], []
    for i, j, _, nonsyn, name in synth.mg94_entries(synth.DEFAULT_THETA, synth.DEFAULT_POSFREQ):
        ei.append(i * 61 + j)
        ef.append(2 * (name in ("AG", "CT")) + int(nonsyn))
    cf = synth.codon_frequencies(synth.DEFAULT_POSFREQ) if col_freq is None else col_freq
    return Template(np.array(ei, dtype=np.int64), np.array(ef, dtype=np.int64), 4, np.asarray(cf, dtype=np.float64), 61)


def gy94_rates(kappa, omega):
    """Formula values of gy94_template per unit branch length."""
    return np.array([1.0, omega, kappa, kappa * omega])


def gtr_template(D, seed):
    """GTR shape for D states: one formula per unordered pair of states, column frequencies pi.  Returns (template,
    exchangeabilities scaled to one expected substitution per unit length)."""
    rng = np.random.default_rng(seed)
    pairs = [(i, j) for i in range(D) for j in range(i + 1, D)]
    ei = [i * D + j for i, j in pairs] + [j * D + i for i, j in pairs]
    ef = list(range(len(pairs))) * 2
    t = Template(np.array(ei, dtype=np.int64), np.array(ef, dtype=np.int64), len(pairs), rng.dirichlet(np.full(D, 5.0)), D)
    x = rng.gamma(1.0, 1.0, size=len(pairs))
    return t, x / -(t.cf * np.diag(t.Q(x))).sum()


def unit_rate(t, x):
    """Formula values x rescaled to one expected substitution per unit length under the template's column frequencies
    (uniform weights for a template without them)."""
    w = np.full(t.D, 1.0 / t.D) if t.cf is None else t.cf
    return np.asarray(x, dtype=np.float64) / -(w * np.diag(t.Q(x))).sum()


def codon_pi(seed):
    """A codon pi of CF3x4 product shape from random position-specific nucleotide frequencies."""
    rng = np.random.default_rng(seed)
    return synth.codon_frequencies(rng.dirichlet(np.full(4, 10.0), size=3))


def workload(D, n_taxa, n_sites, C, mean_t=0.05, seed=20261015):
    """An alignment on a random tree (codon sequences for 61 states, a random reversible model otherwise) whose model is
    replaced by the test's: C rate classes with unequal weights.  Only the tree, leaves, root pi and class weights are used."""
    if D == 61:
        w = synth.codon_workload(n_taxa, n_sites, 1, seed=seed, mean_t=mean_t)
    else:
        w = synth.generic_workload(D, n_taxa, n_sites, 1, seed=seed, mean_t=mean_t)
    w.Q_classes = [np.zeros((D, D))] * C
    cw = np.linspace(1.0, 2.0, C)
    w.class_weights = cw / cw.sum()
    return w


def oracle_P(Q):
    """Transition matrix exp(Q) by the oracle."""
    return port.expm(Q)


def mixture_P(Ms, weights):
    """sum_k w_k exp(M_k): the transition matrix of an explicit-form mixture hand-over."""
    return sum(wk * port.expm(Mk) for wk, Mk in zip(weights, Ms))


def site_lnl(sl, ss):
    return np.log(sl) - 64.0 * np.log(2.0) * ss


def oracle_lnl(w, P, weights=None):
    """(lnL, per-pattern log-likelihoods) of transition matrices P [C, B, D, D] mixed over rate classes with `weights`."""
    wts = w.class_weights if weights is None else weights
    sites = np.stack([site_lnl(*port.prune(w, P[c])) for c in range(P.shape[0])])
    m = sites.max(axis=0)
    site = m + np.log(np.einsum("c,cs->s", np.asarray(wts, dtype=np.float64), np.exp(sites - m)))
    return float((w.pattern_freq * site).sum()), site


def inf_norm(A):
    return float(np.abs(A).sum(axis=1).max())


def p_atol(A, shared_powers=False):
    """Tolerance of a transition matrix against the oracle: 3e-14 while the rate matrix's norm needs no squaring (the
    scaling-and-squaring kernels square above 0.975; the shared-powers polynomial above EXPM_POLY_THETA), 5e-13 above."""
    return 3e-14 if inf_norm(A) <= (EXPM_POLY_THETA if shared_powers else 0.975) else 5e-13
