"""GPU suite (pytest -m gpu): hb2_batch_site_rates, LEISR's site model (one pattern, every branch's rate matrix times the
set's rate) on nucleotide and protein-sized partitions:

  1. the unmodified reference binary's site log-likelihoods at rate 1 (golden fixtures);
  2. the resident path: at rate 1 every pattern equals hb2_evaluate's for its class, every padded size, dense and
     compiled hand-overs;
  3. tests/site_rates_reference.py (long-double exponentials and pruning) over state counts 2..32, rates 1e-3..1e4,
     every tree of tests/test_gpu_shapes.py (the 400-leaf star leaves the double range), ambiguity rows and a
     non-reversible model;
  4. rate 0: identity matrices, log pi_state for constant columns and -inf where no single state explains the column;
  5. chunks: a call spanning two chunks of the stated memory rule equals one-set calls bit for bit;
  6. nothing an evaluation reads is touched;
  7. every refusal, with nothing written.
Root vectors differ from the model's frequencies unless a test says otherwise."""
import numpy as np
import pytest

from hyphy_b200 import synth, LikelihoodFunction, engine
from tests import batch_reference as br
from tests import golden_cases as gc
from tests import site_rates_reference as sr
from tests.test_gpu_shapes import TREES, flat_tree, inject_ambiguity, caterpillar

pytestmark = pytest.mark.gpu

# |got - ref| <= TOL[case] * |ref| per set: ten times the largest error measured on one H100 80GB HBM3 (700 W), rounded
# up to a power of ten (sweep 6.4e-13 at 3 states, shapes 5.7e-13 on the 400-leaf star; the largest errors come from the
# rates whose exponentials need the most squarings).  The resident path at rate 1 measured 2.2e-16.
TOL = {"sweep": 1e-11, "shapes": 1e-11}
RESIDENT_TOL = 1e-13                # against hb2_evaluate's per-pattern values, relative
GOLDEN_SITE_TOL, GOLDEN_LNL_TOL = 1e-9, 1e-10
RATES = [1e-3, 0.01, 0.1, 0.5, 1.0, 2.0, 10.0, 100.0, 1e4]
SWEEP_D = [2, 3, 4, 5, 8, 9, 16, 17, 20, 24, 25, 32]
SWEEP_TREE = [[0, [0, 0]], [0, 0, 0], 0, [0, 0]]          # 9 leaves, a 4-child root, a 3-child node
LENGTHS = np.array([0.02, 0.08, 0.2, 0.5, 1.2])          # branch lengths are drawn from these: few distinct matrices
LONG_LENGTHS = np.array([1.5, 3.0, 6.0])                  # 400-leaf star: every leaf costs several bits
MAX_PATTERNS = 40
RATES_MAX_SETS = 65536                                    # hb2_engine.cu


@pytest.fixture(scope="module", autouse=True)
def _need_gpu(engine_lib):
    assert engine.device_count() > 0, "GPU tests need a CUDA device (no fallback exists)"


# ---------------------------------------------------------------------------------------------------------------------
# workloads
# ---------------------------------------------------------------------------------------------------------------------
def rate_workload(spec, D, seed=0, reversible=True, n_sites=60, amb_frac=0.05, lengths=LENGTHS):
    """(template, workload, root): patterns simulated on the tree under the template's model; ambiguity rows injected."""
    rng = np.random.default_rng(seed + 31 * D)
    tree = flat_tree(spec, seed=seed)
    tree.t = rng.choice(lengths, len(tree.t))
    tree.t[-1] = 0.0
    t = sr.small_template(D, reversible, seed)
    Q = br.dense(t, t.base)
    pi = t.cf if reversible else np.full(D, 1.0 / D)
    Ps = [[np.maximum(synth._expm_np(Q * tree.t[b]), 0.0) for b in range(tree.n_branches)]]
    Ps = [[P / P.sum(axis=1, keepdims=True) for P in Ps[0]]]
    states = synth._simulate(tree, Ps, pi, np.zeros(n_sites, dtype=np.int64), rng)
    ls, freq, s2p = synth.compress(states)
    w = synth.Workload(f"rates{tree.n_leaves}_D{D}", tree, D, pi, [Q], np.array([1.0]), ls, np.zeros((0, D)), freq, s2p,
                       None, {"kind": "generic"})
    if amb_frac:
        inject_ambiguity(w, rng, amb_frac)
    root = np.random.default_rng(seed + 5).dirichlet(np.full(D, 2.0))
    return t, w, root


def rate_sets(w, seed=0, n_random=3):
    """(patterns, rates): every rate of RATES and n_random log-uniform ones, each at up to MAX_PATTERNS patterns
    (the ambiguous ones first)."""
    rng = np.random.default_rng(seed + 99)
    rates = RATES + list(10.0 ** rng.uniform(-3, 2, n_random))
    amb = np.nonzero((w.leaf_states < 0).any(axis=0))[0]
    pats = np.concatenate([amb, np.setdiff1d(np.arange(w.S), amb)])[:MAX_PATTERNS]
    return np.tile(pats, len(rates)), np.repeat(rates, len(pats))


def reference(w, root, pats, rates, mutate=()):
    """Long-double log-likelihoods of the sets, one exponential per distinct (rate, matrix)."""
    A = w.Qt()[0]
    expm = sr.RateExpm()
    out = np.empty(len(pats), dtype=br.LD)
    for r in np.unique(rates):
        sel = np.nonzero(rates == r)[0]
        cols = w.leaf_states[:, pats[sel]].T
        out[sel] = sr.site_lnl(w.tree, A, r, cols, w.ambig, root, expm, mutate)
    return out


def rel_err(got, ref):
    ref = np.asarray(ref, dtype=br.LD)
    return np.asarray(np.abs(np.asarray(got, dtype=br.LD) - ref) / np.abs(ref), dtype=np.float64)


def new_lf(w, handover="dense"):
    lf = LikelihoodFunction(w, flags=engine.FLAG_FORCE_FP64)
    if handover == "dense":
        lf.set_all_matrices()
    else:
        lf.set_template()
        lf.set_all_compiled()
    return lf


def site_lnl(sl, ss):
    return np.log(sl) - 64.0 * np.log(2.0) * ss


def chunk_sets(L, I, D):
    """Sets per chunk of hb2_batch_site_rates (hb2_engine.cu rates_shape): P matrices, node vectors and exponents, rate,
    pattern and result of a set within ~8 GB, at most RATES_MAX_SETS."""
    Dp = sr.pad_states(D)
    per_set = (L + I - 1) * Dp * Dp * 8 + I * (Dp * 8 + 4) + 20
    return min(max(1, int(8.0e9 / per_set)), RATES_MAX_SETS)


# ---------------------------------------------------------------------------------------------------------------------
# 1. reference binary
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["c1_hky85_8x500", "nuc_300x200_scaling"])
def test_golden_at_rate_one(name):
    """HKY85 through its compiled template at rate 1 reproduces the unmodified reference binary's site log-likelihoods."""
    w, g = gc.load(name)
    lf = new_lf(w, "compiled")
    got = lf.part.batch_site_rates(np.arange(w.S), np.ones(w.S), w.pi)
    lf.close()
    assert float(np.abs(got[w.site_to_pattern] - g["site_lnL"]).max()) <= GOLDEN_SITE_TOL
    lnl = float((w.pattern_freq * got).sum())
    assert abs(lnl - g["lnL"]) <= GOLDEN_LNL_TOL * abs(g["lnL"])


# ---------------------------------------------------------------------------------------------------------------------
# 2. resident path
# ---------------------------------------------------------------------------------------------------------------------
RESIDENT = [("nuc", 4), ("rev", 3), ("rev", 7), ("rev", 16), ("rev", 20), ("rev", 29)]     # padded 4, 4, 8, 16, 24, 32


@pytest.mark.parametrize("handover", ["dense", "compiled"])
@pytest.mark.parametrize("kind,D", RESIDENT)
def test_rate_one_matches_resident_path(kind, D, handover):
    """At rate 1 the batch matrices are the resident ones: every pattern equals hb2_evaluate's for its class."""
    w = synth.nucleotide_workload(12, 300, ambig_frac=0.02) if kind == "nuc" else synth.generic_workload(D, 12, 300, n_classes=2)
    lf = new_lf(w, handover)
    S = w.S
    for cat in range(w.C):
        _, sl, ss = lf.part.evaluate(cat, w.pi, want_sites=True)
        ref = site_lnl(sl, ss)
        got = lf.part.batch_site_rates(np.arange(S), np.ones(S), w.pi, cat=cat)
        assert np.all(np.isfinite(got))
        assert float((np.abs(got - ref) / np.abs(ref)).max()) <= RESIDENT_TOL, (cat, float((np.abs(got - ref) / np.abs(ref)).max()))
    lf.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3. long-double reference
# ---------------------------------------------------------------------------------------------------------------------
SWEEP = [(D, True) for D in SWEEP_D] + [(5, False), (20, False)]


@pytest.mark.parametrize("D,reversible", SWEEP)
def test_state_count_sweep(D, reversible):
    t, w, root = rate_workload(SWEEP_TREE, D, seed=1, reversible=reversible)
    pats, rates = rate_sets(w, seed=D)
    lf = new_lf(w)
    got = lf.part.batch_site_rates(pats, rates, root)
    lf.close()
    err = rel_err(got, reference(w, root, pats, rates))
    assert float(err.max()) <= TOL["sweep"], float(err.max())


@pytest.mark.parametrize("D", [4, 20])
@pytest.mark.parametrize("shape", list(TREES))
def test_tree_shapes(shape, D):
    lengths = LONG_LENGTHS if shape == "star400" else LENGTHS
    t, w, root = rate_workload(TREES[shape], D, seed=2, lengths=lengths)
    pats, rates = rate_sets(w, seed=3, n_random=2)
    lf = new_lf(w)
    got = lf.part.batch_site_rates(pats, rates, root)
    lf.close()
    ref = reference(w, root, pats, rates)
    if shape == "star400" and D == 20:
        assert float(np.min(ref)) < -750.0               # some sets' likelihoods lie below the smallest double
    err = rel_err(got, ref)
    assert float(err.max()) <= TOL["shapes"], float(err.max())


# ---------------------------------------------------------------------------------------------------------------------
# 4. rate 0
# ---------------------------------------------------------------------------------------------------------------------
def test_rate_zero():
    """Identity matrices: a column is explained by the states every leaf allows, so lnL = log sum of their root
    frequencies -- log pi_state for a constant column, -inf when none is left.  The value passes through the node
    renormalisation's power of two (log(pi / 2) + log 2), hence the few-ulp bound instead of bit equality."""
    t, w, root = rate_workload(SWEEP_TREE, 5, seed=4, amb_frac=0.1)
    ls = w.leaf_states.copy()
    ls[:, :5] = np.arange(5)[None, :]                    # five constant columns, one per state
    w.leaf_states = ls
    lf = new_lf(w)
    got = lf.part.batch_site_rates(np.arange(w.S), np.zeros(w.S), root)
    lf.close()
    allowed = np.ones((w.S, 5))
    for leaf in range(w.tree.n_leaves):
        codes = ls[leaf]
        rows = np.where(codes[:, None] >= 0, np.arange(5)[None, :] == codes[:, None],
                        w.ambig[np.maximum(-codes - 1, 0)] if len(w.ambig) else 0.0)
        allowed *= rows
    exp = np.log((allowed * root).sum(axis=1), where=allowed.any(axis=1), out=np.full(w.S, -np.inf))
    assert np.array_equal(np.isneginf(got), np.isneginf(exp))
    assert np.isneginf(got).any() and np.isfinite(got).any()
    fin = np.isfinite(exp)
    assert np.all(np.abs(got[fin] - exp[fin]) <= 4 * np.finfo(float).eps * np.abs(exp[fin]))
    assert np.all(np.abs(got[:5] - np.log(root)) <= 4 * np.finfo(float).eps * np.abs(np.log(root)))


def test_rate_beyond_range_is_nan_for_its_set_only():
    t, w, root = rate_workload(SWEEP_TREE, 4, seed=5)
    lf = new_lf(w)
    got = lf.part.batch_site_rates([0, 1, 2], [1.0, 1e300, 0.5], root)
    lf.close()
    assert np.isfinite(got[0]) and np.isnan(got[1]) and np.isfinite(got[2])


# ---------------------------------------------------------------------------------------------------------------------
# 5. chunks
# ---------------------------------------------------------------------------------------------------------------------
def test_chunks_equal_one_set_calls():
    t, w, root = rate_workload(caterpillar(700), 30, seed=6, n_sites=40)
    L, I = w.tree.n_leaves, w.tree.n_internal
    chunk = chunk_sets(L, I, 30)
    n = chunk + 5
    rng = np.random.default_rng(7)
    pats = rng.integers(0, w.S, n)
    rates = 10.0 ** rng.uniform(-2, 1, n)
    lf = new_lf(w)
    lf.compute()                                         # flushes the hand-overs: the launches below are the call's own
    before = lf.part.launch_count
    got = lf.part.batch_site_rates(pats, rates, root)
    assert lf.part.launch_count - before == 4            # two chunks, two kernels each
    one = np.array([lf.part.batch_site_rates(pats[s:s + 1], rates[s:s + 1], root)[0] for s in range(n)])
    lf.close()
    assert np.all(np.isfinite(got))
    assert np.array_equal(got, one)


def test_class_minus_one_is_class_zero():
    w = synth.generic_workload(7, 10, 100, n_classes=2)
    lf = new_lf(w)
    pats, rates = np.arange(w.S), np.linspace(0.1, 3.0, w.S)
    zero = lf.part.batch_site_rates(pats, rates, w.pi, cat=0)
    assert np.array_equal(lf.part.batch_site_rates(pats, rates, w.pi, cat=-1), zero)
    assert not np.array_equal(lf.part.batch_site_rates(pats, rates, w.pi, cat=1), zero)
    lf.close()


# ---------------------------------------------------------------------------------------------------------------------
# 6. no interference
# ---------------------------------------------------------------------------------------------------------------------
def test_no_interference():
    w = synth.generic_workload(20, 16, 200, n_classes=2)
    lf = new_lf(w, "compiled")
    part = lf.part
    part.evaluate(0, w.pi)                               # a branch cache needs every class evaluated
    lnl0, sl0, ss0 = part.evaluate(1, w.pi, want_sites=True)
    cond0 = part.read_conditionals(1, w.tree.n_internal - 1)
    P0 = part.read_transition(1, 3)
    part.branch_cache_build(5, w.pi)
    bc0 = part.branch_cache_evaluate(cat=1, want_sites=False)
    root = np.random.default_rng(8).dirichlet(np.ones(20))
    a = part.batch_site_rates(np.arange(w.S), np.full(w.S, 0.3), root, cat=1)
    b = part.batch_site_rates(np.arange(w.S), np.full(w.S, 0.3), root, cat=1)
    assert np.array_equal(a, b)                          # the resident rate matrices are unchanged
    assert part.branch_cache_evaluate(cat=1, want_sites=False) == bc0
    c1, e1 = part.read_conditionals(1, w.tree.n_internal - 1)
    assert np.array_equal(c1, cond0[0]) and np.array_equal(e1, cond0[1])
    assert np.array_equal(part.read_transition(1, 3), P0)
    lnl1, sl1, ss1 = part.evaluate(1, w.pi, want_sites=True)
    assert lnl1 == lnl0 and np.array_equal(sl1, sl0) and np.array_equal(ss1, ss0)
    lf.close()


# ---------------------------------------------------------------------------------------------------------------------
# 7. refusals
# ---------------------------------------------------------------------------------------------------------------------
def _raw(part, cat, n, pats, rates, root, out):
    """The C entry point with any argument possibly NULL."""
    def ptr(a, t):
        return None if a is None else a.ctypes.data_as(t)
    return part._lib.hb2_batch_site_rates(part._h, cat, n, ptr(pats, engine._ip), ptr(rates, engine._dp), ptr(root, engine._dp),
                                          ptr(out, engine._dp))


def _refused(part, match, *args):
    rc = _raw(part, *args)
    assert rc != 0
    msg = part._lib.hb2_last_error().decode()
    assert match in msg, msg


def test_refusals():
    t, w, root = rate_workload(SWEEP_TREE, 5, seed=9)
    lf = new_lf(w)
    part = lf.part
    lnl = part.evaluate(0, w.pi)
    n = 4
    pats = np.arange(n, dtype=np.int64)
    rates = np.array([0.5, 1.0, 2.0, 0.1])
    out = np.full(n, 7.0)
    bad_pat, neg, nan, inf = pats.copy(), rates.copy(), rates.copy(), rates.copy()
    bad_pat[3] = w.S
    neg[2], nan[1], inf[0] = -0.5, np.nan, np.inf
    cases = [
        (("null argument", 0, n, None, rates, root, out)),
        (("null argument", 0, n, pats, None, root, out)),
        (("null argument", 0, n, pats, rates, None, out)),
        (("null argument", 0, n, pats, rates, root, None)),
        (("nSets=-1 is negative", 0, -1, pats, rates, root, out)),
        (("rate class 1 out of range", 1, n, pats, rates, root, out)),
        ((f"set 3: patternOf={w.S} out of range", 0, n, bad_pat, rates, root, out)),
        (("set 2: rate -0.5 is not a finite number", 0, n, pats, neg, root, out)),
        (("set 1: rate nan is not a finite number", 0, n, pats, nan, root, out)),
        (("set 0: rate inf is not a finite number", 0, n, pats, inf, root, out)),
    ]
    for match, *args in cases:
        _refused(part, match, *args)
        assert np.all(out == 7.0)
    assert part.evaluate(0, w.pi) == lnl
    # branches without a resident rate matrix: a transition matrix, a mixture, none at all
    B = w.tree.n_branches
    P2 = synth._expm_np(w.Qt()[0][2])
    part.set_matrices(0, [2], P2[None], kind=engine.MATRIX_TRANS)
    _refused(part, "rate class 0, branch 2 has no resident rate matrix", 0, n, pats, rates, root, out)
    part.set_matrices(0, [2], w.Qt()[0][2][None])                      # a rate matrix again: accepted
    assert np.all(np.isfinite(part.batch_site_rates(pats, rates, root)))
    Q4 = w.Qt()[0][4]
    part.set_mixture_matrices(0, [4], np.stack([Q4, 2 * Q4])[None], np.array([[0.5, 0.5]]))
    _refused(part, "rate class 0, branch 4 has no resident rate matrix", 0, n, pats, rates, root, out)
    assert np.all(out == 7.0)
    lf.close()
    fresh = LikelihoodFunction(w, flags=engine.FLAG_FORCE_FP64)
    fresh.part.set_matrices(0, np.arange(B - 1), w.Qt()[0][:B - 1])
    _refused(fresh.part, f"rate class 0, branch {B - 1} has no resident rate matrix", 0, n, pats, rates, root, out)
    fresh.part.set_matrices(0, [B - 1], w.Qt()[0][B - 1:])
    assert np.all(np.isfinite(fresh.part.batch_site_rates(pats, rates, root)))
    fresh.close()
    # codon partitions go to hb2_batch_site_likelihoods
    wc, _ = gc.load("mg94_8x60_c1")
    lc = LikelihoodFunction(wc, flags=engine.FLAG_FORCE_FP64)
    lc.set_all_matrices()
    _refused(lc.part, "use hb2_batch_site_likelihoods with formula values multiplied by the rate", 0, 2, pats[:2], rates[:2],
             wc.pi, out[:2].copy())
    lc.close()
    assert np.all(out == 7.0)
