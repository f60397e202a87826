"""Plain high-precision reference of hb2_batch_site_rates (LEISR's site model) for 2..32 states, built on
tests/batch_reference.py's expm_ld and prune_ld:

  * small_template: a sparse rate-matrix template in hb2_set_rate_template's form for any D in 2..32, reversible (column
    frequencies) or not;
  * rate_P: a set's per-branch transition matrices exp(r * A_b) in long double, one exponential per distinct matrix;
  * site_lnl: log-likelihoods of columns at one rate by long-double pruning.

rate_P and site_lnl take `mutate`, a set of labels that each restate one plausible kernel bug (MUTATIONS); the CPU suite
shows that each moves the GPU file's workloads beyond its tolerances.  No test functions live here."""
import numpy as np

from tests import batch_reference as br

LD = br.LD

MUTATIONS = {
    "leaf_only": "the rate multiplies the rate matrices of leaf branches only",
    "rate_twice": "the rate is applied twice (exp(r^2 A))",
    "root_ignored": "the root vector is ignored (uniform root frequencies)",
    "transpose": "every branch's transition matrix is used transposed",
    "amb_off_by_one": "ambiguity code -(r+1) reads row r+1 of the ambiguity table",
    "pad_leak": "an ambiguity leaf also sums the padded states D..Dp-1, each as a matrix entry of one",
}


def pad_states(D):
    return next(p for p in (4, 8, 16, 24, 32, 64) if D <= p)


def small_template(D, reversible=True, seed=0):
    """A br.Template for 2..32 states: every pair of states for D <= 8, else a ring (i, i+1) and chords (i, i + D//3).
    Reversible: one formula per undirected edge and column frequencies; otherwise one formula per direction, none."""
    assert 2 <= D <= 32
    rng = np.random.default_rng(1000 * seed + D + (0 if reversible else 500))
    if D <= 8:
        edges = [(i, j) for i in range(D) for j in range(i + 1, D)]
    else:
        c = D // 3
        edges = [(i, (i + 1) % D) for i in range(D)] + [(i, (i + c) % D) for i in range(D)]
    ei, ef = [], []
    for e, (a, b) in enumerate(edges):
        ei += [a * D + b, b * D + a]
        ef += [e, e] if reversible else [2 * e, 2 * e + 1]
    nF = max(ef) + 1
    base = rng.gamma(2.0, 0.5, nF)
    cf = rng.dirichlet(np.full(D, 5.0)) if reversible else None
    t = br.Template(D, np.array(ei, np.int64), np.array(ef, np.int64), nF, cf, base, np.zeros(nF, np.int64), reversible)
    Q = br.dense(t, base)
    pi = cf if reversible else np.full(D, 1.0 / D)
    t.base = base / -(pi * np.diag(Q)).sum()             # one expected substitution per unit length
    return t


class RateExpm:
    """expm_ld of r * A, computed once per distinct (r, A)."""

    def __init__(self):
        self.memo = {}

    def __call__(self, A, r):
        key = (float(r), np.asarray(A, np.float64).tobytes())
        if key not in self.memo:
            self.memo[key] = br.expm_ld(LD(r) * np.asarray(A, dtype=LD))
        return self.memo[key]


def rate_P(A, r, n_leaves, expm, mutate=()):
    """[B, D, D] long-double transition matrices exp(r A_b) of one set; A [B, D, D] the rate matrices of the class."""
    out = []
    for b, Ab in enumerate(A):
        rb = r
        if "leaf_only" in mutate and b >= n_leaves:
            rb = 1.0
        if "rate_twice" in mutate:
            rb = r * r
        P = expm(Ab, rb)
        out.append(P.T.copy() if "transpose" in mutate else P)
    return np.stack(out)


def site_lnl(tree, A, r, cols, ambig, root, expm=None, mutate=()):
    """Long-double log-likelihoods of columns [n, L] (leaf codes) at rate r under rate matrices A [B, D, D]."""
    expm = RateExpm() if expm is None else expm
    D = A.shape[-1]
    P = rate_P(A, r, tree.n_leaves, expm, mutate)
    amb = np.asarray(ambig, dtype=np.float64)
    if "pad_leak" in mutate and len(amb):
        amb = amb + (pad_states(D) - D)            # rows of P sum to 1: adds Dp - D to every ambiguity leaf's entry
    rt = np.full(D, 1.0 / D) if "root_ignored" in mutate else root
    pm = tuple(m for m in mutate if m == "amb_off_by_one")
    with np.errstate(divide="ignore"):
        return br.prune_ld(tree, P, cols, amb, rt, pm)
