"""Plain high-precision reference of the four batch entry points (hb2_batch_site_likelihoods,
hb2_batch_site_mixture_likelihoods, hb2_batch_column_likelihoods, hb2_batch_site_simulate) for any 33..64-state template:

  * expm_ld: exp(A) by a Taylor series with scaling and squaring in numpy.longdouble (x86-64: 80-bit, u = 2^-64);
  * compact_template: a sparse rate-matrix template with 2D formulas for any D, reversible (column frequencies) or not;
  * set_P: a set's per-branch transition matrices from its formula values and weights, components added in order;
  * prune_ld: Felsenstein's recursion in numpy.longdouble without any scaling, for caller columns with ambiguity rows.

prune_ld and set_P take `mutate`, a set of labels that each restate one plausible kernel bug (MUTATIONS); the CPU suite
shows that each moves the GPU file's workloads beyond its tolerances.  No test functions live here."""
import dataclasses

import numpy as np

LD = np.longdouble
TAYLOR_STOP = LD(2) ** -64          # a term this small against the partial sum ends the series (long double's u)
MAX_TERMS = 40

MUTATIONS = {
    "drop_last": "the last mixture component of every branch with two or more is left out",
    "w0_all": "the weight of component 0 is used for every component of a branch",
    "transpose": "every branch's transition matrix is used transposed",
    "amb_off_by_one": "ambiguity code -(r+1) reads row r+1 of the ambiguity table",
    "pad_leak": "an ambiguity leaf also sums the padded states D..63, each as a matrix entry of one",
    "no_wide_rescale": "fp64 products with one renormalisation per node, none between the children of a wide node",
}


def norm1(A):
    return np.abs(A).sum(axis=-2).max(axis=-1)


def expm_ld(A):
    """exp(A) in long double.  Scaling: X = A / 2^s with the smallest s >= 0 for which ||X||_1 <= 1/2.  Truncation: terms
    X^k / k! are added until one has a 1-norm of at most 2^-64 times the partial sum's; every later term is at most 1/4
    of the one before (||X|| / (k + 1) <= 1/4), so the tail left out is below that term.  Then s squarings."""
    X = np.asarray(A, dtype=LD)
    n = float(norm1(X))
    s = 0 if n <= 0.5 else int(np.ceil(np.log2(n / 0.5)))
    X = X / LD(2) ** s
    S = np.eye(X.shape[0], dtype=LD) + X
    T = X
    for k in range(2, MAX_TERMS):
        T = T @ X / LD(k)
        S = S + T
        if norm1(T) <= TAYLOR_STOP * norm1(S):
            break
    else:
        raise AssertionError("Taylor series did not reach its stopping rule")
    for _ in range(s):
        S = S @ S
    return S


@dataclasses.dataclass
class Template:
    """A rate-matrix template in hb2_set_rate_template's form, with a base rate and a class per formula: a set's
    formula values are base * t_b * (alpha for class 0, beta for class 1), as FEL / MEME scale synonymous and
    nonsynonymous rates."""
    D: int
    ei: np.ndarray                  # flat entry index i * D + j of every entry
    ef: np.ndarray                  # its formula
    nF: int
    cf: np.ndarray | None           # column frequencies (entry (i, j) times cf[j]) or None
    base: np.ndarray                # [nF]
    cls: np.ndarray                 # [nF] 0 or 1
    reversible: bool


def compact_template(D, reversible=True, seed=0):
    """Entries on a ring (i, i+1) and on chords (i, i + D//3), 4D entries and 2D formulas.  Reversible: both directions
    of an undirected edge share its formula and the column frequencies make pi_i q_ij symmetric.  Non-reversible: forward
    and backward directions have their own formulas (ring and chord of one start state share), no column frequencies,
    so exp(Qt) and its transpose give different likelihoods."""
    assert 33 <= D <= 64
    rng = np.random.default_rng(1000 * seed + D + (0 if reversible else 500))
    c = D // 3
    ei, ef = [], []
    for e, (a, b) in enumerate([(i, (i + 1) % D) for i in range(D)] + [(i, (i + c) % D) for i in range(D)]):
        if reversible:
            fa = fb = e
        else:
            fa, fb = e % D, D + e % D
        ei += [a * D + b, b * D + a]
        ef += [fa, fb]
    nF = 2 * D
    base = rng.gamma(2.0, 0.5, nF)
    cls = (np.arange(nF) % 3 == 0).astype(np.int64)
    cf = rng.dirichlet(np.full(D, 5.0)) if reversible else None
    t = Template(D, np.array(ei, np.int64), np.array(ef, np.int64), nF, cf, base, cls, reversible)
    Q = dense(t, base)
    pi = cf if reversible else np.full(D, 1.0 / D)
    t.base = base / -(pi * np.diag(Q)).sum()             # one expected substitution per unit length
    return t


def dense(t, v, dtype=np.float64):
    """Rate matrix of one row of formula values: scatter, column frequencies, diagonal = minus the row sum."""
    M = np.zeros((t.D, t.D), dtype=dtype)
    M.flat[t.ei] = np.asarray(v, dtype=dtype)[t.ef]
    if t.cf is not None:
        M *= np.asarray(t.cf, dtype=dtype)[None, :]
    M[np.diag_indices(t.D)] = 0
    M[np.diag_indices(t.D)] = -M.sum(axis=1)
    return M


def row_values(t, length, scale_syn, scale_nonsyn):
    return t.base * length * np.where(t.cls == 1, scale_nonsyn, scale_syn)


class ExpmCache:
    """exp of the rate matrix of one row of formula values, by `fn` (expm_ld, or the oracle's fp64 expm), computed once
    per distinct row."""

    def __init__(self, t, fn):
        self.t, self.fn, self.memo = t, fn, {}

    def __call__(self, v):
        key = np.asarray(v, dtype=np.float64).tobytes()
        if key not in self.memo:
            if self.fn is expm_ld:
                self.memo[key] = expm_ld(dense(self.t, v, LD))
            else:
                self.memo[key] = np.asarray(self.fn(dense(self.t, v)), dtype=LD)
        return self.memo[key]


def set_P(expm, V, W, branch_k, mutate=()):
    """Per-branch matrices [B, D, D] (long double) of one set: rows V [R, nF], weights W [R] (None: one row per branch,
    no weights), components of a branch consecutive and added in component order."""
    out, r = [], 0
    for m in branch_k:
        if W is None:
            acc = expm(V[r])
        else:
            wts = [W[r]] * m if "w0_all" in mutate else list(W[r:r + m])
            used = m - 1 if ("drop_last" in mutate and m > 1) else m
            acc = LD(wts[0]) * expm(V[r])
            for c in range(1, used):
                acc = acc + LD(wts[c]) * expm(V[r + c])
        out.append(acc.T.copy() if "transpose" in mutate else acc)
        r += m
    return np.stack(out)


def prune_ld(tree, P, cols, ambig, root, mutate=()):
    """log-likelihoods (long double) of columns [n, L] (leaf codes: state >= 0, ambiguity row -(r+1)) under P [B, D, D]
    and the root vector, by tests/resident_reference.py's recursion without scaling (80-bit exponents reach 2^-16382).
    'pad_leak' adds 64 - D to every entry of every ambiguity row: each entry of the leaf's vector grows by 64 - D times
    its matrix row sum, which is one -- the 64 - D padded states, each as a matrix entry of one."""
    from tests import resident_reference as rr          # it builds on this module's expm_ld
    if "no_wide_rescale" in mutate:
        return _prune_fp64_node_scaled(tree, P, cols, ambig, root)
    amb = np.asarray(ambig, dtype=LD)
    if "amb_off_by_one" in mutate and len(amb):
        amb = np.roll(amb, -1, axis=0)                      # code -(r+1) reads row (r+1) mod nAmb
    if "pad_leak" in mutate:
        amb = amb + LD(64 - P.shape[-1])
    return rr.class_sites(tree, P, cols, amb, root)


def _prune_fp64_node_scaled(tree, P, cols, ambig, root):
    """The 'no_wide_rescale' mutation: fp64 throughout, each node's vector brought to max 1 (exponent kept) only once its
    children are all multiplied in."""
    cols = np.atleast_2d(np.asarray(cols, dtype=np.int64))
    n, L, D = len(cols), tree.n_leaves, P.shape[-1]
    Pd = np.asarray(P, dtype=np.float64)
    amb = np.asarray(ambig, dtype=np.float64)
    cond, ex = [None] * tree.n_internal, [None] * tree.n_internal
    for i, kids in enumerate(tree.children()):
        v, e = np.ones((n, D)), np.zeros(n)
        for c in kids:
            if c < L:
                codes = cols[:, c]
                m = np.where((codes >= 0)[:, None], Pd[c][:, np.maximum(codes, 0)].T,
                             (amb[np.maximum(-codes - 1, 0)] @ Pd[c].T) if len(amb) else 0.0)
            else:
                m = cond[c - L] @ Pd[c].T
                e = e + ex[c - L]
            v = v * m
        mx = v.max(axis=1)
        k = np.where(mx > 0, np.floor(np.log2(np.where(mx > 0, mx, 1.0))) + 1, 0)
        cond[i], ex[i] = v * np.exp2(-k)[:, None], e + k
    with np.errstate(divide="ignore"):
        return np.log(cond[-1] @ np.asarray(root, dtype=np.float64)) + ex[-1] * np.log(2.0)
