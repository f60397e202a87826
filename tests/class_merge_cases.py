"""Exact reference for the rate-class merge L_s = sum_c w_c L_{c,s} and its log, and builders for the workloads that
probe it at the edges: classes far apart in scale, zero and tiny weights, impossible patterns.  No test functions live
here; tests/test_class_merge_reference.py pins these on the CPU.

The per-class likelihoods come in the reference's convention L = siteL * 2^(-64 * siteScale).  The sum is formed in
exact rationals, so no class underflows or is cut, and a class of weight 0 takes no part at all, as the reference skips
such a class (likefunc2.cpp:668).  The oracle's own merge (hb2o_combine) cannot serve here: it aligns on class 0 whatever
its weight, and its 2^64-step scaler underflows in exactly these cases."""
import math
from fractions import Fraction

import numpy as np

from hyphy_b200 import synth

# ln 2 split so that k * LN2_HI is exact for |k| < 2^20 (fdlibm's constants)
LN2_HI = 6.93147180369123816490e-01
LN2_LO = 1.90821492927058770002e-10


def exact_log(x: Fraction) -> float:
    """log(x) of a rational to an ulp or two: x = r * 2^k with r in (1/2, 2), log(float(r)) + k ln 2 summed exactly."""
    if x == 0:
        return -math.inf
    if x < 0:
        return math.nan
    k = x.numerator.bit_length() - x.denominator.bit_length()
    r = x / Fraction(2) ** k
    # float(r) rounds once (r in (1/2, 2)); logs of its numerator and denominator would cancel thousands of bits
    return math.fsum([math.log(float(r)), k * LN2_HI, k * LN2_LO])


def exact_class_sum(site_l, site_scale, weights, s) -> Fraction | None:
    """sum_c w_c siteL[c,s] 2^(-64 siteScale[c,s]) as a rational; None if a class of weight != 0 (or a weight) is NaN."""
    tot = Fraction(0)
    for c in range(len(weights)):
        wc = float(weights[c])
        if wc == 0.0:
            continue
        lc = float(site_l[c][s])
        if math.isnan(wc) or math.isnan(lc):
            return None
        tot += Fraction(wc) * Fraction(lc) * Fraction(2) ** (-64 * int(site_scale[c][s]))
    return tot


def exact_site_lnl(site_l, site_scale, weights) -> np.ndarray:
    """Per-pattern log sum_c w_c siteL[c] 2^(-64 siteScale[c]) (siteL, siteScale: [C, S]); classes of weight 0 are
    skipped, NaN in a class of weight != 0 gives NaN, no positive class gives -inf."""
    site_l = np.asarray(site_l, dtype=np.float64)
    site_scale = np.asarray(site_scale, dtype=np.int64)
    assert site_l.shape == site_scale.shape and site_l.shape[0] == len(weights)
    out = np.empty(site_l.shape[1])
    for s in range(site_l.shape[1]):
        tot = exact_class_sum(site_l, site_scale, weights, s)
        out[s] = math.nan if tot is None else exact_log(tot)
    return out


def exact_lnl(site, freq) -> float:
    """sum_s f_s site_s over the patterns with f_s > 0 (math.fsum); -inf if any of them is -inf, NaN if any is NaN."""
    terms = [float(f) * float(x) for f, x in zip(freq, site) if f > 0]
    if any(math.isnan(t) for t in terms):
        return math.nan
    if any(t == -math.inf for t in terms):
        return -math.inf
    return math.fsum(terms)


def engine_site_lnl(site_l, site_scale) -> np.ndarray:
    """log(siteL * 2^(-64 siteScale)) of the engine's per-pattern outputs, with no rounding of its own."""
    return exact_site_lnl(np.asarray(site_l)[None], np.asarray(site_scale)[None], [1.0])


def class_exponents(site_l, site_scale) -> np.ndarray:
    """log2 of each per-class likelihood ([C, S]); -inf where it is 0."""
    with np.errstate(divide="ignore"):
        return np.log2(np.asarray(site_l, dtype=np.float64)) - 64.0 * np.asarray(site_scale, dtype=np.float64)


# Tolerances of the GPU checks against the oracle: (lnL rtol, per-pattern atol).  fp64: 1e-10 / 1e-8.  Tensor path
# (D > 32): 1e-7 / 1e-5, but the 3xTF32 split carries a matrix entry to about 2^-22 relative, and on the stacks below, with
# one entry on every branch, that error has the same sign everywhere and adds up along the tree; so the per-pattern bound
# grows with it, 1e-4 at 400 branches (the merge faults these cases catch are -inf, NaN or errors far above it).
def tolerances(w, mode):
    if mode == "tc" and w.D > 32:
        return 1e-7, max(1e-5, 2.5e-7 * w.tree.n_branches)
    return 1e-10, 1e-8


# ---------------------------------------------------------------------------------------------------------------------
# Dense transition-matrix stacks (MATRIX_TRANS hand-overs), [B, D, D] per class

def identity(B, D):
    """P = I on every branch: a constant pattern of state k has L = pi_k at the root, any other pattern L = 0."""
    return np.broadcast_to(np.eye(D), (B, D, D)).copy()


def flat(B, D, x):
    """Every entry x ("scaled rows"; x = 1/D is a uniform-row matrix).  A leaf's message is x, an internal node's is x * D
    times its own (equal) entries, so any pattern has L = x^B * D^(I-1) * sum(pi) on a tree of B branches, I internal
    nodes."""
    return np.full((B, D, D), float(x))


def uniform(B, D):
    return flat(B, D, 1.0 / D)


def flat_log2(tree, D, x):
    """log2 L of a flat class under a root vector summing to 1."""
    return tree.n_branches * math.log2(x) + (tree.n_internal - 1) * math.log2(D)


def flat_below_identity(tree, D, bits):
    """The entry x of a flat stack whose class sits `bits` below an identity class (log2 L = -log2 D on a constant
    pattern) under a uniform root vector; negative bits put it above."""
    return 2.0 ** (-(bits + tree.n_internal * math.log2(D)) / tree.n_branches)


def class_stack(spec, tree, D):
    """'identity', 'uniform', ('below', bits) or ('flat', x)."""
    B = tree.n_branches
    if spec == "identity":
        return identity(B, D)
    if spec == "uniform":
        return uniform(B, D)
    kind, v = spec
    if kind == "below":
        return flat(B, D, flat_below_identity(tree, D, v))
    assert kind == "flat"
    return flat(B, D, v)


def flat_entry(spec, tree, D):
    """x of a flat class spec."""
    if spec == "uniform":
        return 1.0 / D
    return flat_below_identity(tree, D, spec[1]) if spec[0] == "below" else spec[1]


# ---------------------------------------------------------------------------------------------------------------------
# Alignments

def constant_workload(D, n_leaves, S, C, seed=20261016, n_free=0, zero_freq=(), weights=None, pi=None):
    """S patterns on a random binary tree with n_leaves leaves.  All are constant (every leaf in one random state)
    except the last n_free, whose leaves take random states (never all equal).  Frequencies are 1..3, 0 for the
    patterns listed in zero_freq.  The root vector is uniform unless given.  The C classes' matrices are handed over by
    the test; Q_classes only carries the class count."""
    rng = np.random.default_rng(seed + 7 * D + n_leaves)
    tree = synth.random_tree(n_leaves, seed + n_leaves)
    leaf = np.tile(rng.integers(0, D, size=S), (n_leaves, 1))
    for s in range(S - n_free, S):
        col = rng.integers(0, D, size=n_leaves)
        col[1] = (col[0] + 1) % D
        leaf[:, s] = col
    freq = rng.integers(1, 4, size=S).astype(np.int64)
    freq[list(zero_freq)] = 0
    pi = np.full(D, 1.0 / D) if pi is None else np.asarray(pi, dtype=np.float64)
    wts = np.full(C, 1.0 / C) if weights is None else np.asarray(weights, dtype=np.float64)
    return synth.Workload(f"const{D}_{n_leaves}x{S}_c{C}", tree, D, pi, [np.zeros((D, D))] * C, wts, leaf.astype(np.int64),
                          np.zeros((0, D)), freq, np.arange(S, dtype=np.int64), None, {"kind": "generic"})


def is_constant(w):
    return (w.leaf_states == w.leaf_states[0]).all(axis=0)


# The scale-gap workloads of tests/test_gpu_class_merge.py: (D, leaves, class specs, the range in bits that class 0 sits
# above class 1 on every constant pattern).  tests/test_class_merge_reference.py checks each range against the oracle.
GAP_CASES = {
    "d61_identity_uniform": (61, 200, ("identity", "uniform"), (1100, 1200)),
    "d20_identity_uniform": (20, 260, ("identity", "uniform"), (1100, 1130)),
    "d4_identity_uniform": (4, 600, ("identity", "uniform"), (1190, 1200)),
    "d61_three": (61, 200, ("identity", "uniform", ("below", 1200)), (1100, 1200)),
    "d61_gap990": (61, 200, ("identity", ("below", 990)), (985, 995)),
    "d61_gap1010": (61, 200, ("identity", ("below", 1010)), (1001, 1020)),
    "d61_gap1030": (61, 200, ("identity", ("below", 1030)), (1025, 1035)),
    "d61_gap1062": (61, 200, ("identity", ("below", 1062)), (1055, 1070)),
    "d61_gap500": (61, 200, ("identity", ("below", 500)), (495, 505)),
    "d61_gap1100": (61, 200, ("identity", ("below", 1100)), (1095, 1105)),
    "d61_gap3000": (61, 200, ("identity", ("below", 3000)), (2995, 3005)),
    "d61_above": (61, 200, ("identity", ("below", -400)), (-405, -395)),     # class 1 has L = 2^394 > 1
}


def gap_case(name, S=300, n_free=0, zero_freq=(), weights=None, pi=None, order=None):
    """(workload, P[C, B, D, D]) of a GAP_CASES entry; `order` permutes the classes (and `weights` is in that order)."""
    D, n_leaves, specs, _ = GAP_CASES[name]
    if order is not None:
        specs = tuple(specs[i] for i in order)
    w = constant_workload(D, n_leaves, S, len(specs), n_free=n_free, zero_freq=zero_freq, weights=weights, pi=pi)
    return w, np.stack([class_stack(sp, w.tree, D) for sp in specs])
