"""Plain high-precision reference of the resident evaluation path (hb2_evaluate, hb2_evaluate_classes,
hb2_evaluate_forced, the branch cache, hb2_read_conditionals and hb2_read_transition), built on
tests/batch_reference.py's expm_ld:

  * Expm: exp of a handed-over rate matrix in numpy.longdouble, computed once per distinct matrix;
  * class_sites: Felsenstein's recursion in long double without any scaling (x86-64: 80-bit, exponents down to 2^-16382)
    for one rate class -- ambiguity rows, any root vector, optionally one node pinned to a state per pattern, and the
    conditionals of every internal node as row-normalised vectors;
  * merge: the class merge log sum_c w_c L_c over the classes of non-zero weight;
  * evaluate: per-class and merged per-pattern log-likelihoods of a set of matrices;
  * substitute: the matrix the shared-powers expm stage exponentiates for a batch entry, given its group's reference.

evaluate and substitute take `mutate`, a set of labels that each restate one plausible kernel bug (MUTATIONS); the CPU
suite shows that each moves the GPU file's workloads beyond its tolerances.  No test functions live here."""
import numpy as np

from tests import batch_reference as br

LD = br.LD
SHARE_TOL = 1e-13             # hb2_kernels_fp64.cuh, expm_classify_kernel: the proportionality bound

MUTATIONS = {
    "share_proportionality": "an entry is taken for its group's direction times the weight ratio when every value's share "
                             "of the weight matches the reference's to 1e-13 (a bound on the share, not on the value)",
    "fp32_root": "the root vector is staged through float",
    "fp32_class_weights": "the class weights are staged through float",
}


class Expm:
    """expm_ld of a float64 matrix, computed once per distinct matrix."""

    def __init__(self):
        self.memo = {}

    def __call__(self, A):
        A = np.ascontiguousarray(A, dtype=np.float64)
        key = A.tobytes()
        if key not in self.memo:
            self.memo[key] = br.expm_ld(A.astype(LD))
        return self.memo[key]


def class_sites(tree, P, cols, ambig, root, pin=None, want_cond=False):
    """Log-likelihoods (long double) [n] of columns [n, L] (leaf codes: state >= 0, ambiguity row -(r+1)) under one rate
    class's matrices P [B, D, D] and the root vector.  pin = (flat node id, states [n]): a pinned leaf shows that state,
    a pinned internal node keeps only that state's entry.  want_cond: also the conditionals of every internal node
    [I][n, D], each row divided by its maximum (rows that are all zero stay zero)."""
    cols = np.atleast_2d(np.asarray(cols, dtype=np.int64))
    n, L, D = len(cols), tree.n_leaves, P.shape[-1]
    Pl = np.asarray(P, dtype=LD)
    amb = np.asarray(ambig, dtype=LD)
    node, states = pin if pin is not None else (-1, None)
    cond = [None] * tree.n_internal
    for i, kids in enumerate(tree.children()):
        v = np.ones((n, D), dtype=LD)
        for c in kids:
            if c < L:
                codes = np.asarray(states, dtype=np.int64) if c == node else cols[:, c]
                obs = codes >= 0
                m = np.empty((n, D), dtype=LD)
                m[obs] = Pl[c][:, codes[obs]].T                         # (P x)[k] = P[k][state]
                if not obs.all():
                    m[~obs] = amb[-codes[~obs] - 1] @ Pl[c].T
            else:
                m = cond[c - L] @ Pl[c].T
            v = v * m
        if L + i == node:
            keep = np.zeros((n, D), dtype=LD)
            keep[np.arange(n), states] = 1
            v = v * keep
        cond[i] = v
    with np.errstate(divide="ignore"):
        lnl = np.log(cond[-1] @ np.asarray(root, dtype=LD))
    if not want_cond:
        return lnl
    norm = []
    for v in cond:
        mx = v.max(axis=1, keepdims=True)
        norm.append(v / np.where(mx > 0, mx, 1))
    return lnl, norm


def merge(per_class, weights):
    """log sum_c w_c exp(l_c) [n] over the classes with w_c > 0 (a zero-weight class never enters, even at -inf)."""
    w = np.asarray(weights, dtype=LD)
    keep = w > 0
    lc = np.asarray(per_class, dtype=LD)[keep]
    m = lc.max(axis=0)
    safe = np.where(np.isfinite(m), m, 0)
    with np.errstate(divide="ignore"):
        return safe + np.log((w[keep][:, None] * np.exp(lc - safe)).sum(axis=0))


def evaluate(tree, P, cols, ambig, root, weights, mutate=()):
    """(merged [n], per_class [C, n]) log-likelihoods of columns [n, L] under matrices P [C, B, D, D]."""
    if "fp32_root" in mutate:
        root = np.asarray(root, dtype=np.float32)
    if "fp32_class_weights" in mutate:
        weights = np.asarray(weights, dtype=np.float32)
    per = np.stack([class_sites(tree, P[c], cols, ambig, root) for c in range(len(P))])
    return merge(per, weights), per


def share_flagged(v, v_ref):
    """The classification by shares of the weight: |v_k w_ref - v_ref w_k| <= 1e-13 w_k w_ref for every value."""
    v, vr = np.asarray(v, dtype=np.float64).ravel(), np.asarray(v_ref, dtype=np.float64).ravel()
    wk, wr = np.abs(v).sum(), np.abs(vr).sum()
    return bool(np.all(np.abs(v * wr - vr * wk) <= SHARE_TOL * wk * wr))


def value_flagged(v, v_ref):
    """The classification by values: |v_k w_ref - v_ref w_k| <= 1e-13 |v_ref| w_k for every value."""
    v, vr = np.asarray(v, dtype=np.float64).ravel(), np.asarray(v_ref, dtype=np.float64).ravel()
    wk, wr = np.abs(v).sum(), np.abs(vr).sum()
    return bool(np.all(np.abs(v * wr - vr * wk) <= SHARE_TOL * np.abs(vr) * wk))


def substitute(A, A_ref, v=None, v_ref=None, mutate=()):
    """The rate matrix exponentiated for a shared-powers entry A whose group's reference is A_ref; v, v_ref are the values
    classified (formula values of a compiled hand-over; None: the dense matrices themselves).  Without mutation that is A.
    'share_proportionality': the reference direction times the weight ratio wherever share_flagged holds."""
    if "share_proportionality" not in mutate:
        return A
    v = A if v is None else v
    v_ref = A_ref if v_ref is None else v_ref
    if not share_flagged(v, v_ref):
        return A
    return np.asarray(A_ref, dtype=np.float64) * (np.abs(v).sum() / np.abs(v_ref).sum())
