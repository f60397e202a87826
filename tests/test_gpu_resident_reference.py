"""GPU suite (pytest -m gpu): the resident evaluation path against tests/resident_reference.py (long-double exponentials
and pruning) at the precision the fp64 path exists for.  The oracle suites (test_gpu_shapes.py, test_gpu_parity.py,
test_gpu_sequences.py) hold these kernels to 1e-10 of lnL and 1e-8 per pattern; here every family is held to ten times
the largest error measured on an H100, so a kernel that loses a few digits fails.

  1. kernel families x state counts: every padded size of the small-state walk and DMMA kernels, the fp64 lanes kernel
     and the tensor walk at 33..64 states, non-reversible models; four rate classes (one of weight 0), pattern
     frequencies above 1, dense and compiled hand-overs: lnL, every pattern, every class, pinned nodes, the branch cache,
     conditionals and transition matrices;
  2. the exponentials' switch points: lengths on both sides of every scaling and degree step, relative steps of 1e-9;
  3. near-proportional inputs on the shared-powers path, classified against a reference in the batch and against the
     cached direction;
  4. every tree of test_gpu_shapes.TREES and its wide-node underflow workloads;
  5. pattern counts at the edges of the pattern tiles, and the split-pairs walk under HB2_WALK_LANES=1.
Every workload has a Dirichlet root vector other than the model's frequencies and ambiguity rows (the all-ones row
among them).  Likelihoods, pinned nodes and conditionals are checked against long-double pruning of the matrices the
partition reports (read_transition), and those matrices against expm_ld entry by entry.  The two are kept apart because
an fp64 exponential, the oracle's included, is accurate to about 1e-16 of the row, not of the entry: at 64 states a
ring template puts entries near 1e-34, some off by several per cent, and a pattern pinned to an unlikely state runs
through them (1e-4 relative on the 64-state sweep, reproduced with the oracle's exponential on the CPU).  The largest error of each family and measure is printed at the end of the module (pytest -s)."""
import copy
import dataclasses

import numpy as np
import pytest

from hyphy_b200 import synth, LikelihoodFunction, engine
from tests import batch_reference as br
from tests import resident_reference as rr
from tests import sequence_cases as sc
from tests import site_rates_reference as sr
from tests.test_gpu_shapes import TREES, UNDERFLOW, expected_kernel, flat_tree, inject_ambiguity, pad_states, underflow_workload

pytestmark = pytest.mark.gpu

# Largest |got - ref| / |ref| per pattern ("site"), relative lnL error ("lnl"), |got - ref| per transition-matrix entry
# ("matrix"; "matrix_sq" for the small-state switch lengths with five squarings or more, see many_squarings) and per
# row-normalised conditional ("cond": relative on entries >= 2^-40 of the row maximum, absolute below that), per kernel
# family: ten times the largest value measured on one H100 80GB HBM3 (700 W), rounded up to a power of ten.  Measured
# (site / lnl / matrix / matrix_sq / cond): small walk 2.3e-16 / 1.8e-16 / 1.4e-15 / 2.2e-13 / 1.2e-15, small DMMA
# 2.8e-16 / 1.9e-16 / 4.3e-15 / 1.7e-13 / 2.2e-15, fp64 lanes 1.8e-16 / 2.1e-16 / 2.3e-15 / - / 4.2e-15, tensor walk
# 1.4e-7 / 7.3e-9 / 2.3e-15 (the fp64 exponential) / - / 2.4e-6.  The many-squaring lengths (norms 2^4..2^6 and a
# saturating one) lose two digits to the squarings; every other length is held to the tighter bound.
# The workloads hand the shared-powers path exact scalings only, which its classification accepts to rounding; an
# entry it accepts may differ from the direction it is evaluated as by 1e-13 of every value, 1e-13 ||A||_inf in P.
TOL = {
    "small_walk": {"site": 1e-14, "lnl": 1e-14, "matrix": 1e-13, "matrix_sq": 1e-11, "cond": 1e-13},
    "small_dmma": {"site": 1e-14, "lnl": 1e-14, "matrix": 1e-13, "matrix_sq": 1e-11, "cond": 1e-13},
    "lanes": {"site": 1e-14, "lnl": 1e-14, "matrix": 1e-13, "cond": 1e-13},
    "tc": {"site": 1e-5, "lnl": 1e-7, "matrix": 1e-13, "cond": 1e-4},
}
LENGTHS = np.array([0.02, 0.08, 0.2, 0.5, 1.2])          # branch lengths are drawn from these: few distinct matrices
RATES = np.array([0.3, 0.8, 1.4, 2.6])                    # four rate classes ...
WEIGHTS = np.array([0.3, 0.0, 0.45, 0.25])                # ... one of weight 0
SWEEP_TREE = [[0, [0, 0]], [0, 0, 0], [[0, 0], [0, 0, 0]], 0, [0, [0, 0]], [0, 0]]   # 17 leaves, 26 branches (>= 24)
COND_FLOOR = 2.0 ** -40

MEASURED = {}
TC_BIAS = []


@pytest.fixture(scope="module", autouse=True)
def _need_gpu(engine_lib):
    assert engine.device_count() > 0, "GPU tests need a CUDA device (no fallback exists)"
    yield
    for (fam, what), v in sorted(MEASURED.items()):
        print(f"resident-reference max {fam:10s} {what:7s} {v:.3e}")
    for case, signed, mean in TC_BIAS:
        print(f"resident-reference tc bias {case}: signed lnL {signed:+.3e}, mean |site| {mean:.3e}")


def family(D, mode):
    Dp = pad_states(D)
    return "tc" if (mode == "tc" and Dp == 64) else "lanes" if Dp == 64 else "small_dmma" if Dp >= 16 else "small_walk"


def within(fam, what, err, info=""):
    err = float(err)
    MEASURED[fam, what] = max(MEASURED.get((fam, what), 0.0), err)
    assert err <= TOL[fam][what], (fam, what, err, info)


def rel(got, ref):
    ref = np.asarray(ref, dtype=rr.LD)
    return np.asarray(np.abs(np.asarray(got, dtype=rr.LD) - ref) / np.abs(ref), dtype=np.float64)


def site_lnl(sl, ss):
    return np.log(np.asarray(sl, dtype=rr.LD)) - rr.LD(64) * np.log(rr.LD(2)) * np.asarray(ss, dtype=rr.LD)


# ---------------------------------------------------------------------------------------------------------------------
# workloads
# ---------------------------------------------------------------------------------------------------------------------
NONREV = {4: lambda: sc.nrm_Q(4), 20: lambda: sc.random_Q(20, 20), 48: lambda: sc.random_Q(48, 48),
          64: lambda: sc.drift_Q(64, 64)}


def model(D, reversible=True):
    """(br.Template, stationary vector): small_template / compact_template, or a generic template (every off-diagonal
    entry its own formula) holding one of tests/sequence_cases.py's non-reversible generators."""
    if reversible:
        t = sr.small_template(D) if D <= 32 else br.compact_template(D)
        return t, t.cf
    Q, pi = NONREV[D]()
    g = sc.generic_template(D)
    return br.Template(D, g.ei, g.ef, g.nF, None, sc.offdiag(Q), np.zeros(g.nF, np.int64), False), pi


class Case:
    """A workload and what it hands over: template t, rates[c] * lengths[b] * t.base as formula values (compiled) or
    their dense rate matrices, the root vector, and the long-double matrices of the reference."""

    def __init__(self, spec, D, reversible=True, S=200, rates=RATES, weights=WEIGHTS, seed=0, lengths=LENGTHS):
        rng = np.random.default_rng(seed + 31 * D)
        self.expm = rr.Expm()
        self.t, pi = model(D, reversible)
        tree = flat_tree(spec, seed=seed)
        tree.t = rng.choice(lengths, len(tree.t))
        tree.t[-1] = 0.0
        self.rates, self.D = np.asarray(rates, dtype=np.float64), D
        Q = br.dense(self.t, self.t.base)
        Ps = [[self.expm(Q * tree.t[b]).astype(np.float64) for b in range(tree.n_branches)]]
        Ps = [[np.maximum(P, 0) / np.maximum(P, 0).sum(axis=1, keepdims=True) for P in Ps[0]]]
        states = synth._simulate(tree, Ps, pi, np.zeros(4 * S + 400, dtype=np.int64), rng)
        ls, _, _ = synth.compress(states)
        ls = ls[:, :S].copy()                              # at most S patterns (a 3-leaf tree has fewer)
        freq = rng.integers(1, 6, ls.shape[1])
        self.w = synth.Workload(f"resident_D{D}", tree, D, pi, [Q * r for r in self.rates], np.asarray(weights, np.float64),
                                ls, np.zeros((0, D)), freq, np.arange(ls.shape[1]), None, {"kind": "generic"})
        inject_ambiguity(self.w, rng)
        self.root = rng.dirichlet(np.full(D, 2.0))
        self.w.pi = self.root                              # what LikelihoodFunction hands over as the root vector
        self._P = None

    @property
    def tree(self):
        return self.w.tree

    def values(self, c, scale=1.0):
        """Formula values [B, nF] of class c."""
        return self.t.base[None, :] * (self.rates[c] * self.tree.t[:self.tree.n_branches] * scale)[:, None]

    def dense(self, c, scale=1.0):
        return np.stack([br.dense(self.t, v) for v in self.values(c, scale)])

    def P(self):
        """[C, B, D, D] long-double transition matrices."""
        if self._P is None:
            self._P = np.stack([np.stack([self.expm(A) for A in self.dense(c)]) for c in range(len(self.rates))])
        return self._P

    def engine_P(self, lf):
        """[C, B, D, D] the transition matrices the partition holds, in long double: the likelihood checks prune these,
        so they measure the pruning kernels; the exponentials are held to expm_ld entry by entry (check_matrices)."""
        return np.stack([np.stack([lf.part.read_transition(c, b) for b in range(self.tree.n_branches)])
                         for c in range(len(self.rates))]).astype(rr.LD)

    def head(self, S):
        """The same case restricted to its first S patterns (matrices and their exponentials shared)."""
        c = copy.copy(self)
        c.w = dataclasses.replace(self.w, leaf_states=self.w.leaf_states[:, :S].copy(),
                                  pattern_freq=self.w.pattern_freq[:S].copy(), site_to_pattern=np.arange(S))
        return c

    def cols(self):
        return self.w.leaf_states.T

    def open(self, mode, handover="dense"):
        lf = LikelihoodFunction(self.w, flags=engine.FLAG_FORCE_FP64 if mode == "fp64" else engine.FLAG_DEFAULT)
        assert lf.part.pruning_kernel in expected_kernel(self.D, mode), lf.part.pruning_kernel
        if handover == "dense":
            for c in range(len(self.rates)):
                lf.part.set_matrices(c, lf.all_nodes, self.dense(c))
        else:
            lf.part.set_rate_template(self.t.ei, self.t.ef, self.t.nF, self.t.cf)
            for c in range(len(self.rates)):
                lf.part.set_matrices_compiled(c, lf.all_nodes, self.values(c))
        return lf


# ---------------------------------------------------------------------------------------------------------------------
# shared checks
# ---------------------------------------------------------------------------------------------------------------------
def check_merged(case, lf, fam, label=""):
    """lnL and every pattern of hb2_evaluate_classes; returns the reference's per-class values."""
    merged, per = rr.evaluate(case.tree, case.engine_P(lf), case.cols(), case.w.ambig, case.root, case.w.class_weights)
    lnl, sl, ss = lf.part.evaluate_classes(case.w.class_weights, case.root, want_sites=True)
    ref = (case.w.pattern_freq * merged).sum()
    assert np.isfinite(lnl)
    within(fam, "lnl", rel(lnl, ref), label)
    err = rel(site_lnl(sl, ss), merged)
    within(fam, "site", err.max(), label)
    if fam == "tc":
        TC_BIAS.append((f"D{case.D} S{case.w.S} {label}", float((lnl - ref) / abs(ref)), float(err.mean())))
    return per


def check_classes(case, lf, fam, per):
    for c in range(len(case.rates)):
        lnl, sl, ss = lf.part.evaluate(c, case.root, want_sites=True)
        within(fam, "site", rel(site_lnl(sl, ss), per[c]).max(), f"class {c}")
        within(fam, "lnl", rel(lnl, (case.w.pattern_freq * per[c]).sum()), f"class {c}")


def check_matrices(case, lf, fam, classes=None):
    P = case.P()
    for c in (range(len(case.rates)) if classes is None else classes):
        for b in range(case.tree.n_branches):
            within(fam, "matrix", np.abs(lf.part.read_transition(c, b) - P[c, b]).max(), (c, b))


def check_forced(case, lf, fam, nodes, unlikely_node=None, c=2):
    """Pinned nodes: random states, and at unlikely_node every pattern's least likely state."""
    rng = np.random.default_rng(case.D)
    P = case.engine_P(lf)[c]
    todo = [(n, rng.integers(0, case.D, case.w.S)) for n in nodes]
    if unlikely_node is not None:
        _, cond = rr.class_sites(case.tree, P, case.cols(), case.w.ambig, case.root, want_cond=True)
        todo.append((unlikely_node, np.argmin(cond[unlikely_node - case.tree.n_leaves], axis=1)))
    for node, fs in todo:
        ref = rr.class_sites(case.tree, P, case.cols(), case.w.ambig, case.root, pin=(node, fs))
        lnl, sl, ss = lf.part.evaluate_forced(c, case.root, node, fs)
        ok = np.isfinite(ref)
        assert np.array_equal(sl > 0, ok), node
        within(fam, "site", rel(site_lnl(sl[ok], ss[ok]), ref[ok]).max(), f"forced {node}")
        if ok.all():
            within(fam, "lnl", rel(lnl, (case.w.pattern_freq * ref).sum()), f"forced {node}")


def check_branch_cache(case, lf, fam, node):
    """Branch cache built under the case's root vector; the branch's matrix of every class replaced by its length x 2.5
    = a full long-double recomputation with the new matrices."""
    lf.part.evaluate_classes(case.w.class_weights, case.root)
    lf.part.branch_cache_build(node, case.root)
    for c in range(len(case.rates)):
        A = br.dense(case.t, case.values(c, 2.5)[node])
        lf.part.set_matrices(c, [node], A[None])
    lnl, sl, ss = lf.part.branch_cache_evaluate(case.w.class_weights, want_sites=True)
    P = case.engine_P(lf)
    for c in range(len(case.rates)):
        within(fam, "matrix", np.abs(P[c, node] - case.expm(br.dense(case.t, case.values(c, 2.5)[node]))).max(), "cache")
    merged, _ = rr.evaluate(case.tree, P, case.cols(), case.w.ambig, case.root, case.w.class_weights)
    within(fam, "lnl", rel(lnl, (case.w.pattern_freq * merged).sum()), f"cache {node}")
    within(fam, "site", rel(site_lnl(sl, ss), merged).max(), f"cache {node}")
    for c in range(len(case.rates)):
        lf.part.set_matrices(c, [node], case.dense(c)[node][None])
    lf.part.evaluate_classes(case.w.class_weights, case.root, update_nodes=[node])


def cond_err(got, ref):
    """Row-normalised conditionals: relative on entries >= 2^-40 of the row maximum, absolute (to the maximum) below."""
    mx = got.max(axis=1, keepdims=True)
    g = np.asarray(got / np.where(mx > 0, mx, 1), dtype=rr.LD)
    big = ref >= COND_FLOOR
    e = np.where(big, np.abs(g - ref) / np.where(big, ref, 1), np.abs(g - ref))
    return float(np.asarray(e, dtype=np.float64).max())


def check_conditionals(case, lf, fam, c=0):
    lf.part.evaluate(c, case.root)
    _, cond = rr.class_sites(case.tree, case.engine_P(lf)[c], case.cols(), case.w.ambig, case.root, want_cond=True)
    for inode in range(case.tree.n_internal):
        got, _ = lf.part.read_conditionals(c, inode)
        within(fam, "cond", cond_err(got, cond[inode]), inode)


def widest_node(tree):
    ch = tree.children()
    i = int(np.argmax([len(c) for c in ch]))
    return tree.n_leaves + i, ch[i][0]


# ---------------------------------------------------------------------------------------------------------------------
# 1. kernel families x state counts
# ---------------------------------------------------------------------------------------------------------------------
SMALL_D = [2, 3, 4, 5, 8, 9, 16, 17, 20, 24, 25, 32]
WIDE_D = [33, 40, 47, 48, 49, 61, 63, 64]
SWEEP = ([(D, "fp64", True) for D in SMALL_D] + [(D, m, True) for D in WIDE_D for m in ("fp64", "tc")]
         + [(4, "fp64", False), (20, "fp64", False)] + [(D, m, False) for D in (48, 64) for m in ("fp64", "tc")])
_CASES = {}


def sweep_case(D, reversible):
    key = ("sweep", D, reversible)
    if key not in _CASES:
        _CASES[key] = Case(SWEEP_TREE, D, reversible, S=min(200, 60 if D == 2 else 200), seed=1)
    return _CASES[key]


@pytest.mark.parametrize("D,mode,reversible", SWEEP)
def test_state_count_sweep(D, mode, reversible):
    case = sweep_case(D, reversible)
    fam = family(D, mode)
    L, I = case.tree.n_leaves, case.tree.n_internal
    lf = case.open(mode, "dense")
    per = check_merged(case, lf, fam, "dense")
    check_classes(case, lf, fam, per)
    check_matrices(case, lf, fam)
    node, under = widest_node(case.tree)
    check_forced(case, lf, fam, [0, L + I // 2, L + I - 1], unlikely_node=node)
    check_branch_cache(case, lf, fam, under)
    check_conditionals(case, lf, fam)
    lf.close()
    lf = case.open(mode, "compiled")
    check_merged(case, lf, fam, "compiled")
    check_matrices(case, lf, fam, classes=[0, 3])
    lf.close()


# ---------------------------------------------------------------------------------------------------------------------
# 2. switch points of the exponentials
# ---------------------------------------------------------------------------------------------------------------------
def row_norm(A):
    return np.abs(A).sum(axis=1).max()


def many_squarings(label):
    """The small-state switch lengths whose exponentials take five squarings or more (norms from 2^4 up, saturating):
    their matrices are held to the "matrix_sq" bound, every other matrix of the small families to "matrix"."""
    return label == "saturating" or label.split()[0] in ("16", "32", "64")


def switch_lengths(Q, kind):
    """(label, length) pairs that put ||Q t||_inf on both sides of every switch of the exponential, 1e-9 apart."""
    n = row_norm(Q)
    if kind == "small":               # expm_small_kernel: s = binary exponent of the largest row norm
        marks = [2.0 ** k for k in range(7)]
        extra = [("saturating", 4000.0 / n)]
    elif kind == "dmma":              # expm64_dmma_kernel: Paterson-Stockmeyer degree steps of ||A|| / 2^s
        marks = [0.0064, 0.069, 0.245, 0.55, 0.975, 2 * 0.55, 2 * 0.975, 8 * 0.975]
        extra = []
    else:                             # expm_poly_kernel: rho = 2.3 * 2^s
        marks = [2.3, 4.6, 9.2]
        extra = [("rho 1e-8", 1e-8 / n), ("zero", 0.0)]
    out = []
    for m in marks:
        out += [(f"{m:g} below", m * (1 - 1e-9) / n), (f"{m:g} above", m * (1 + 1e-9) / n)]
    return out + extra


@pytest.mark.parametrize("kind,D,handover", [("small", D, "dense") for D in (2, 4, 5, 8, 16, 20, 32)]
                         + [("dmma", D, "dense") for D in (48, 64)]
                         + [("poly", D, h) for D in (48, 61, 64) for h in ("dense", "compiled")])
def test_expm_switch_points(kind, D, handover, monkeypatch):
    """Class 0 holds the switch-point matrices on its first branches (the poly batch opens with an ordinary length: the
    group's reference; every entry is proportional to it, so all go through the polynomial).  Every matrix against
    expm_ld, entry by entry, and every pattern of class 0."""
    if kind == "dmma":
        monkeypatch.setenv("HB2_EXPM_SHARED", "0")
    case = Case(SWEEP_TREE, D, rates=[1.0], weights=[1.0], S=100, seed=2)
    fam = family(D, "fp64")
    Q = br.dense(case.t, case.t.base)
    lens = switch_lengths(Q, kind)
    if kind == "poly":
        lens = [("reference", 0.3)] + lens
    B = case.tree.n_branches
    assert len(lens) <= B
    t = case.tree.t.copy()
    t[:len(lens)] = [x for _, x in lens]
    case.tree.t = t
    lf = case.open("fp64", handover)
    P = case.P()
    for b, (label, x) in enumerate(lens):
        got = lf.part.read_transition(0, b)
        if label == "zero":
            assert np.array_equal(got, np.eye(D))
            continue
        within(fam, "matrix_sq" if many_squarings(label) else "matrix", np.abs(got - P[0, b]).max(), label)
    lnl, sl, ss = lf.part.evaluate(0, case.root, want_sites=True)
    ref = rr.class_sites(case.tree, case.engine_P(lf)[0], case.cols(), case.w.ambig, case.root)
    within(fam, "site", rel(site_lnl(sl, ss), ref).max(), kind)
    if kind == "poly":
        # the polynomial really served the batch: the product kernel alone rounds every such matrix differently
        served = [b for b, (label, _) in enumerate(lens) if label not in ("zero", "rho 1e-8")]
        shared = [lf.part.read_transition(0, b) for b in served]
        lf.close()
        monkeypatch.setenv("HB2_EXPM_SHARED", "0")
        lf = case.open("fp64", handover)
        for b, got in zip(served, shared):
            assert not np.array_equal(got, lf.part.read_transition(0, b)), lens[b][0]
    lf.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3. near-proportional inputs on the shared-powers path
# ---------------------------------------------------------------------------------------------------------------------
SHARE_MOVES = [0.5e-13, 0.9e-13, 1.1e-13, 1e-12, 1e-10]


def near_proportional(A, v, move, compiled):
    """(values', smallest-share index): the value with the smallest nonzero share of the weight moved so that its share
    changes by `move`.  Dense input (v = A flattened): its row's diagonal takes the opposite change, rows still sum to 0."""
    v = np.asarray(v, dtype=np.float64).copy()
    w = np.abs(v).sum()
    cand = np.nonzero(v > 0)[0]
    if not compiled:
        D = A.shape[0]
        cand = cand[cand // D != cand % D]
    f = cand[np.argmin(v[cand])]
    if compiled:                                       # (v + d) / (w + d) - v / w = move
        d = move * w * w / (w - v[f] - move * w)
        v[f] += d
    else:                                              # (v + d) / (w + 2d) - v / w = move
        d = move * w * w / (w - 2 * v[f] - 2 * move * w)
        i = f // A.shape[0]
        v[f] += d
        v[i * A.shape[0] + i] -= d
    return v, f


def probe_pattern(case, leaf, i, j):
    """A column in which `leaf` shows state j and every other leaf state i: its likelihood runs through P_leaf[i, j]."""
    col = np.full(case.tree.n_leaves, i, dtype=np.int64)
    col[leaf] = j
    return col


@pytest.mark.parametrize("route", ["in_batch", "cached"])
@pytest.mark.parametrize("handover", ["dense", "compiled"])
@pytest.mark.parametrize("D", [48, 61, 64])
def test_near_proportional_inputs(D, handover, route, monkeypatch):
    """Branch 1 (a leaf) of class 0 gets a matrix whose smallest-share value is moved off its group's direction.  In the
    batch: handed over with the whole class (entry 0, proportional, is the group's reference).  Cached: handed over alone
    after the whole class built the group's table (classified against the cached direction).  Its exponential must be
    expm_ld of the matrix actually handed over (an entry taken for the direction misses it by 1e-13 of the weight, some
    1e-13 absolute in P), and the probe pattern through that entry must be the pruning of the matrices held."""
    case = Case(SWEEP_TREE, D, rates=[1.0], weights=[1.0], S=100, seed=3)
    fam = family(D, "fp64")
    compiled = handover == "compiled"
    leaf = 1
    case.tree.t[leaf] = LENGTHS[-1]                    # the longest length: the largest move in P per move in the rates
    A0 = case.dense(0)
    V0 = case.values(0)
    other = 2                                          # a proportional branch handed over beside the moved one
    monkeypatch.setenv("HB2_EXPM_SHARED", "0")
    lf = case.open("fp64", handover)
    product_only = lf.part.read_transition(0, other)
    lf.close()
    monkeypatch.delenv("HB2_EXPM_SHARED")
    for move in SHARE_MOVES:
        src = V0[leaf] if compiled else A0[leaf].ravel()
        v, f = near_proportional(A0[leaf], src, move, compiled)
        A = br.dense(case.t, v) if compiled else v.reshape(D, D)
        if compiled:
            e = np.nonzero(case.t.ef == f)[0][0]
            i, j = divmod(int(case.t.ei[e]), D)
        else:
            i, j = divmod(int(f), D)
        w = case.w
        w.leaf_states[:, 0] = probe_pattern(case, leaf, i, j)
        lf = LikelihoodFunction(w, flags=engine.FLAG_FORCE_FP64)
        assert lf.part.pruning_kernel in expected_kernel(D, "fp64"), lf.part.pruning_kernel
        if compiled:
            lf.part.set_rate_template(case.t.ei, case.t.ef, case.t.nF, case.t.cf)
            rows = V0.copy()
            if route == "in_batch":
                rows[leaf] = v
            lf.part.set_matrices_compiled(0, lf.all_nodes, rows)
            lf.part.evaluate(0, case.root)
            if route == "cached":
                lf.part.set_matrices_compiled(0, [leaf, other], np.stack([v, V0[other]]))
        else:
            rows = A0.copy()
            if route == "in_batch":
                rows[leaf] = A
            lf.part.set_matrices(0, lf.all_nodes, rows)
            lf.part.evaluate(0, case.root)
            if route == "cached":
                lf.part.set_matrices(0, [leaf, other], np.stack([A, A0[other]]))
        _, sl, ss = lf.part.evaluate(0, case.root, want_sites=True)
        P = case.engine_P(lf)[0]
        lf.close()
        # the shared-powers path served the batch: the proportional neighbour came from the polynomial (the product
        # kernel alone rounds it differently), in the cached route after classification against the cached direction
        assert not np.array_equal(np.asarray(P[other], dtype=np.float64), product_only), (move, route)
        within(fam, "matrix", np.abs(P[leaf] - case.expm(A)).max(), (move, route))
        ref = rr.class_sites(case.tree, P, w.leaf_states.T, w.ambig, case.root)
        within(fam, "site", rel(site_lnl(sl, ss), ref).max(), (move, route))


# ---------------------------------------------------------------------------------------------------------------------
# 4. tree shapes
# ---------------------------------------------------------------------------------------------------------------------
SHAPE_MODES = [(4, "fp64"), (20, "fp64"), (48, "fp64"), (48, "tc"), (61, "fp64"), (61, "tc")]


def shape_case(shape, D):
    key = ("shape", shape, D)
    if key not in _CASES:
        _CASES[key] = Case(TREES[shape], D, rates=[1.0], weights=[1.0], S=60, seed=len(shape),
                           lengths=np.array([1.5, 3.0]) if shape == "star400" else LENGTHS)
    return _CASES[key]


@pytest.mark.parametrize("D,mode", SHAPE_MODES)
@pytest.mark.parametrize("shape", list(TREES))
def test_tree_shapes(shape, D, mode):
    case = shape_case(shape, D)
    fam = family(D, mode)
    lf = case.open(mode)
    check_merged(case, lf, fam, shape)
    node, under = widest_node(case.tree)
    check_forced(case, lf, fam, [], unlikely_node=node, c=0)
    check_branch_cache(case, lf, fam, under)
    lf.close()


@pytest.mark.parametrize("name,mode", [(n, m) for n in UNDERFLOW for m in (["fp64", "tc"] if UNDERFLOW[n][1] > 32 else ["fp64"])])
def test_wide_node_underflow(name, mode):
    """Stars whose products over the root's children fall below 2^-1022 before the end of the node."""
    w = underflow_workload(name)
    root = np.random.default_rng(7).dirichlet(np.full(w.D, 2.0))
    lf = LikelihoodFunction(w, flags=engine.FLAG_FORCE_FP64 if mode == "fp64" else engine.FLAG_DEFAULT)
    assert lf.part.pruning_kernel in expected_kernel(w.D, mode), lf.part.pruning_kernel
    lf.set_all_matrices()
    lnl, sl, ss = lf.part.evaluate(0, root, want_sites=True)
    P = np.stack([lf.part.read_transition(0, b) for b in range(w.tree.n_branches)]).astype(rr.LD)
    lf.close()
    ref = rr.class_sites(w.tree, P, w.leaf_states.T, w.ambig, root)
    assert float(np.min(ref)) < -750.0
    fam = family(w.D, mode)
    within(fam, "lnl", rel(lnl, (w.pattern_freq * ref).sum()), name)
    within(fam, "site", rel(site_lnl(sl, ss), ref).max(), name)


# ---------------------------------------------------------------------------------------------------------------------
# 5. pattern counts at the tile edges
# ---------------------------------------------------------------------------------------------------------------------
TILE_S = [1, 2, 31, 32, 33, 127, 128, 129, 255, 256, 257, 383, 384, 385]


@pytest.mark.parametrize("S", TILE_S)
@pytest.mark.parametrize("D,mode", [(4, "fp64"), (20, "fp64"), (48, "fp64"), (48, "tc")])
def test_tile_edges(D, mode, S):
    """S = 129 on the tensor walk: a two-tile unit whose second tile holds one pattern, so its warpgroup runs ahead of the
    other through the side-product steps.  Before those steps awaited their ring phase, a warpgroup could restage a
    ring slot the other still read, and this case gave 2.4e-4 of lnL in most evaluations."""
    key = ("tile", D)
    if key not in _CASES:
        _CASES[key] = Case(SWEEP_TREE, D, S=max(TILE_S), seed=4)
    case = _CASES[key].head(S)
    assert case.w.S == S
    lf = case.open(mode)
    check_merged(case, lf, family(D, mode), f"S={S}")
    lf.close()


@pytest.mark.parametrize("mode", ["fp64", "tc"])
def test_split_pairs_one_lane(mode, monkeypatch):
    """HB2_WALK_LANES=1: one lane per (class, tile), every split pair of the walk on it."""
    monkeypatch.setenv("HB2_WALK_LANES", "1")
    case = shape_case("poly33", 48)
    lf = case.open(mode)
    check_merged(case, lf, family(48, mode), "lanes=1")
    lf.close()
