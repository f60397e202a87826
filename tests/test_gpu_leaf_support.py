"""GPU suite (pytest -m gpu): hb2_batch_leaf_support, every leaf's predictive state distribution given the other leaves
(ReconstructAncestors(MARGINAL, DOLEAVES), MEME's and PRIME's --impute-states), against the unmodified reference binary's
fixtures, the long-double reference (tests/leaf_support_reference.py), the oracle's forced-column brute force, and the
device's own brute force through hb2_batch_column_likelihoods:

  1. the reference binary's rows: bsrel_12x80_k3 (mixture layout, K = 3 on every branch) and mg94_8x60_c1 (plain);
  2. every state count 33..64 where the kernels change behaviour, reversible and not, plain sets and mixture sets with
     branchK taking 1..4 in one set, ambiguity rows; fp64 and default partitions bit-identical;
  3. the caller's root vector: Dirichlet, uniform, sparse, and zeros (NaN rows, a -inf site);
  4. every tree shape of tests/test_gpu_shapes.py at 48 states, leaves under the root and the 400-leaf star included;
  5. identities: plain sets = unit-weight mixtures bit for bit, siteLnL = the likelihood entry points bit for bit, a row
     does not move when its own leaf's code changes;
  6. the oracle brute force (port.expm, port.prune per forced column) on 8-taxon workloads with ambiguity, and the
     device brute force (one column per leaf and state through hb2_batch_column_likelihoods);
  7. NaN weights and formula values confined to their set; chunks of more than 1024 sets; repeated calls;
  8. non-interference with evaluations, the branch cache and the other batch entry points' workspace; every refusal
     (class-group mode needs two ranks: tests/test_multigpu.py's territory, not exercised here).

Every call checks that siteLnL equals the likelihood entry point's for the same arguments bit for bit."""
import functools
import re

import numpy as np
import pytest

from hyphy_b200 import LikelihoodFunction, synth, engine
from hyphy_b200.engine import _check, _d, _i, _dp
from oracle import port
from tests import batch_reference as br
from tests import golden_cases as gc
from tests import leaf_support_reference as lsr
from tests import test_gpu_branch_rows_shapes as GS
from tests.test_gpu_batch_mixture import LF, meme_sets, site_lnl, with_omegas
from tests.test_gpu_batch_shapes import SWEEP, expm_for, new_lf, shape_case, sweep_case
from tests.test_gpu_branch_rows import CodonExpm
from tests.test_gpu_shapes import TREES, flat_tree, star, tree_workload

pytestmark = pytest.mark.gpu

# |got - ref| <= TOL_ABS per entry and <= TOL_REL * ref on entries >= BIG, against the long-double reference: ten times
# the largest error measured on one H100 80GB HBM3 (700 W), rounded up to a power of ten.  Measured: 9.4e-16 absolute and
# 5.6e-15 relative over the sweep, root and small-tree cases; 3.1e-14 and 4.1e-13 on the 400-leaf star and the 700-leaf
# caterpillar (LARGE_*, the trees of 100 branches or more)
TOL_ABS, TOL_REL = 1e-14, 1e-13
LARGE_ABS, LARGE_REL = 1e-12, 1e-11
BIG = 1e-6
FIX_TOL = 1e-9                      # absolute, against the reference binary's printed rows (measured: 1.7e-15)
BRUTE_TOL = 1e-11                   # relative on entries >= BIG, against the device and oracle brute forces (4.5e-15)
SUM_TOL = 1e-13                     # |sum_k row[k] - 1|
FIXTURES = {"bsrel_12x80_k3": True, "mg94_8x60_c1": False}      # name: mixture layout
SWEEP_LEAVES = SWEEP + [(33, False), (64, False)]


@pytest.fixture(scope="module", autouse=True)
def _need_gpu(engine_lib):
    assert engine.device_count() > 0, "GPU tests need a CUDA device (no fallback exists)"


# ---------------------------------------------------------------------------------------------------------------------
# workloads, calls and references
# ---------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def sweep_support_case(D, reversible, mix):
    """The batch-shapes sweep workload (9 leaves, a 4-child root, a 3-child node, ambiguity rows, a Dirichlet root),
    plain or K = 4 with branchK 1..4, and its long-double exponentials (shared between tests: treat as read-only)."""
    if mix:
        return GS.sweep_rows_case(D, reversible)
    case = sweep_case(D, reversible, False)
    return case, br.ExpmCache(case.tmpl, br.expm_ld)


@functools.lru_cache(maxsize=None)
def shape_support_case(shape, mix):
    case = shape_case(shape, 48, mix)
    return case, expm_for(case)


def fixture_sets(w):
    """A fixture's model as one set: (V [R, nF], W [R] or None, branch_k [B])."""
    nb = w.tree.n_branches
    mix = w.meta.get("mixture")
    if mix is None:
        return with_omegas(w, w.meta["omegas"]).compiled_values()[0], None, np.ones(nb, np.int64)
    K = len(mix["omegas"])
    comp = with_omegas(w, mix["omegas"]).compiled_values()                   # [K, B, nF]
    return comp.transpose(1, 0, 2).reshape(nb * K, -1), np.tile(mix["weights"], nb), np.full(nb, K, np.int64)


def support_call(lf, case, V=None, W=None, root=None, pats=None, bg=None):
    """(support, site) of a batch-shapes Case, and siteLnL checked against the likelihood entry point bit for bit."""
    V = case.V if V is None else V
    W = (case.W if case.mix else None) if W is None else W
    root = case.root if root is None else root
    pats = case.pats if pats is None else pats
    bk = case.branch_k if W is not None else None
    sup, site = lf.part.batch_leaf_support(pats, V, root, weights=W, branch_k=bk, branch_group=bg, want_site=True)
    if W is None:
        want = lf.part.batch_site_likelihoods(pats, V, root, branch_group=bg)
    else:
        want = lf.part.batch_site_mixture_likelihoods(pats, V, W, root, branch_k=bk, branch_group=bg)
    assert np.array_equal(site, want, equal_nan=True)
    return sup, site


def ref_support(case, expm, sets, V=None, W=None, root=None, outside=False):
    """Long-double rows [len(sets), L, D]: the brute force, or the outside pass (`outside`)."""
    V = case.V if V is None else V
    W = (case.W if case.mix else None) if W is None else W
    root = case.root if root is None else root
    fn = lsr.outside_support if outside else lsr.brute_support
    return np.stack([fn(case.w.tree, expm, V[s], None if W is None else W[s], case.branch_k,
                        case.w.leaf_states[:, case.pats[s]], case.w.ambig, root) for s in sets])


def errors(got, ref):
    """(max absolute error, max relative error on entries >= BIG)."""
    ref = np.asarray(ref, dtype=br.LD)
    err = np.abs(np.asarray(got, dtype=br.LD) - ref)
    big = np.abs(ref) >= BIG
    return float(err.max()), float((err[big] / np.abs(ref[big])).max())


def check_support(got, ref, label, tol_abs=TOL_ABS, tol_rel=TOL_REL):
    assert np.all(np.isfinite(got)), label
    ea, er = errors(got, ref)
    s = float(np.abs(got.sum(axis=-1) - 1).max())
    print(f"[{label}] max |got - ref| = {ea:.2e}, relative on entries >= {BIG:g}: {er:.2e}, |row sum - 1| {s:.2e}")
    assert ea <= tol_abs and er <= tol_rel, (label, ea, er)
    assert s <= SUM_TOL, (label, s)
    return ea, er


def normalise(lnl):
    """Rows [.., D] from forced-column log-likelihoods."""
    x = np.exp(lnl - lnl.max(axis=-1, keepdims=True))
    return x / x.sum(axis=-1, keepdims=True)


# ---------------------------------------------------------------------------------------------------------------------
# 1. the reference binary's rows
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(FIXTURES))
def test_fixture_matches_reference(name):
    """Every site of the fixture (tools/make_golden.py --impute), one set per pattern."""
    w, g0 = gc.load(name)
    g = np.load(gc.GOLDEN_DIR + f"/{name}_impute.npz")
    assert str(g["checksum"]) == gc.checksum(w)
    V, W, branch_k = fixture_sets(w)
    assert (W is not None) == FIXTURES[name]
    pats = np.arange(w.S)
    lf = LF(w)
    Vs = np.ascontiguousarray(np.broadcast_to(V, (w.S,) + V.shape))
    Ws = None if W is None else np.ascontiguousarray(np.broadcast_to(W, (w.S,) + W.shape))
    sup, site = lf.part.batch_leaf_support(pats, Vs, w.pi, weights=Ws, branch_k=None if W is None else branch_k,
                                           want_site=True)
    lf.close()
    assert np.abs(site[w.site_to_pattern] - g0["site_lnL"]).max() <= 1e-9
    err = np.abs(sup[w.site_to_pattern] - g["support"]).max()
    print(f"[fixture {name}] max |got - reference binary| = {err:.2e}")
    assert err <= FIX_TOL


# ---------------------------------------------------------------------------------------------------------------------
# 2. state counts
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D,reversible", SWEEP_LEAVES, ids=[f"{d}{'' if r else '-nonrev'}" for d, r in SWEEP_LEAVES])
def test_state_sweep(D, reversible):
    for mix in (False, True):
        case, expm = sweep_support_case(D, reversible, mix)
        if mix:
            assert set(case.branch_k) == {1, 2, 3, 4}
        src = case.w.leaf_states[:, case.pats]
        assert (src < 0).any() and (src == -1).any()
        out = {}
        for flags in (engine.FLAG_FORCE_FP64, engine.FLAG_DEFAULT):
            lf = new_lf(case, flags)
            out[flags] = support_call(lf, case)
            lf.close()
        sup, site = out[engine.FLAG_FORCE_FP64]
        assert np.array_equal(sup, out[engine.FLAG_DEFAULT][0]) and np.array_equal(site, out[engine.FLAG_DEFAULT][1])
        check_support(sup, ref_support(case, expm, range(case.n)), f"sweep D={D} rev={reversible} mix={mix}")


# ---------------------------------------------------------------------------------------------------------------------
# 3. the caller's root vector
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mix", [False, True], ids=["plain", "mix"])
def test_root_vectors(mix):
    case, expm = sweep_support_case(48, False, mix)
    D = case.w.D
    rng = np.random.default_rng(48)
    sparse = np.zeros(D)
    keep = rng.permutation(D)[:D - D // 3]
    sparse[keep] = rng.dirichlet(np.full(len(keep), 2.0))
    roots = {"dirichlet": case.root, "uniform": np.full(D, 1.0 / D), "sparse": sparse}
    lf = new_lf(case)
    got = {}
    for name, root in roots.items():
        got[name], _ = support_call(lf, case, root=root)
        check_support(got[name], ref_support(case, expm, range(case.n), root=root), f"root {name} mix={mix}")
    assert np.median(np.abs(got["dirichlet"] - got["uniform"])) > 1e3 * TOL_ABS
    sup, site = support_call(lf, case, root=np.zeros(D))
    lf.close()
    assert np.all(np.isnan(sup)) and np.all(site == -np.inf)


# ---------------------------------------------------------------------------------------------------------------------
# 4. tree shapes
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", list(TREES))
def test_tree_shapes(shape):
    for mix in (False, True):
        case, expm = shape_support_case(shape, mix)
        L = case.w.tree.n_leaves
        lf = new_lf(case)
        sup, site = support_call(lf, case)
        lf.close()
        if shape == "star400":
            assert np.all(site < -1022 * np.log(2.0))                       # the product leaves the double range
        assert any(c < L for c in case.w.tree.children()[-1]) or shape in ("all_internal", "bifurcating_root")
        big = case.w.tree.n_branches >= 100
        sets = range(2) if big else range(case.n)
        tol = (LARGE_ABS, LARGE_REL) if big else (TOL_ABS, TOL_REL)
        check_support(sup[list(sets)], ref_support(case, expm, sets, outside=big), f"shape {shape} mix={mix}", *tol)


# ---------------------------------------------------------------------------------------------------------------------
# 5. identities
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D,reversible", [(33, False), (61, True), (64, True)], ids=["33-nonrev", "61", "64"])
def test_plain_equals_unit_weight_mixture(D, reversible):
    case, _ = sweep_support_case(D, reversible, False)
    lf = new_lf(case)
    plain, site_p = support_call(lf, case)
    B = case.w.tree.n_branches
    ones = np.ones((case.n, B))
    mixed, site_m = lf.part.batch_leaf_support(case.pats, case.V, case.root, weights=ones, branch_k=np.ones(B, np.int64),
                                               want_site=True)
    lf.close()
    assert np.array_equal(plain, mixed) and np.array_equal(site_p, site_m)


@pytest.mark.parametrize("mix", [False, True], ids=["plain", "mix"])
def test_row_ignores_own_code(mix):
    """A second partition whose leaf l holds other codes (a state, ambiguity rows) at every pattern: row l of every set
    is bit-identical; the other leaves' rows move."""
    case, _ = sweep_support_case(48, False, mix)
    w = case.w
    lf = new_lf(case)
    base, _ = support_call(lf, case)
    lf.close()
    for l, codes in ((0, 5), (4, -1), (w.tree.n_leaves - 1, -len(w.ambig))):
        ls = w.leaf_states.copy()
        ls[l] = codes
        w2 = synth.Workload(w.name, w.tree, w.D, w.pi, w.Q_classes, w.class_weights, ls, w.ambig, w.pattern_freq,
                            w.site_to_pattern, None, w.meta)
        lf = LikelihoodFunction(w2, flags=engine.FLAG_FORCE_FP64)
        lf.part.set_rate_template(case.tmpl.ei, case.tmpl.ef, case.tmpl.nF, case.tmpl.cf)
        got = lf.part.batch_leaf_support(case.pats, case.V, case.root, weights=case.W if mix else None,
                                         branch_k=case.branch_k if mix else None)
        lf.close()
        assert np.array_equal(got[:, l], base[:, l]), l
        others = np.arange(w.tree.n_leaves) != l
        assert not np.array_equal(got[:, others], base[:, others]), l


# ---------------------------------------------------------------------------------------------------------------------
# 6. brute forces: the oracle and the device
# ---------------------------------------------------------------------------------------------------------------------
def oracle_brute(w, col, P):
    """[L, D] by port.prune of every forced column under the fp64 matrices P."""
    cols = lsr.forced_columns(col, w.D)
    n = len(cols)
    wf = synth.Workload("forced", w.tree, w.D, w.pi, w.Q_classes, w.class_weights, np.ascontiguousarray(cols.T), w.ambig,
                        np.ones(n, np.int64), np.arange(n))
    sl, ss = port.prune(wf, P)
    with np.errstate(divide="ignore"):
        return normalise(site_lnl(sl, ss).reshape(w.tree.n_leaves, w.D))


@pytest.mark.parametrize("mix", [False, True], ids=["plain", "mix"])
def test_oracle_brute_force(mix):
    w, _ = gc.load("mg94_8x60_c4_ambig")
    rng = np.random.default_rng(31 + mix)
    n = 4
    branch_k, V, W, _ = meme_sets(w, 3, n, rng)
    if not mix:                                       # one row per branch: component 0 of every branch
        off = np.concatenate([[0], np.cumsum(branch_k)])
        V, W, branch_k = V[:, off[:-1]], None, np.ones(w.tree.n_branches, np.int64)
    amb = np.nonzero((w.leaf_states < 0).any(axis=0))[0]
    pats = np.concatenate([amb[:2], rng.choice(w.S, n - 2, replace=False)])
    lf = LF(w)
    sup, site = lf.part.batch_leaf_support(pats, V, w.pi, weights=W, branch_k=branch_k if mix else None, want_site=True)
    lf.close()
    ex = CodonExpm(w, False)
    for s in range(n):
        P = np.asarray(br.set_P(ex, V[s], None if W is None else W[s], branch_k), dtype=np.float64)
        want = oracle_brute(w, w.leaf_states[:, pats[s]], P)
        _, er = errors(sup[s], want)
        assert er <= BRUTE_TOL and np.abs(sup[s] - want).max() <= 1e-13, (s, er)


def device_brute(lf, case, sets, W=None):
    """[len(sets), L, D] by hb2_batch_column_likelihoods: one column per (leaf, state), normalised."""
    L, D = case.w.tree.n_leaves, case.w.D
    W = (case.W if case.mix else None) if W is None else W
    out = []
    for s in sets:
        cols = lsr.forced_columns(case.w.leaf_states[:, case.pats[s]], D)
        Vs = np.repeat(case.V[s:s + 1], len(cols), axis=0)
        Ws = None if W is None else np.repeat(W[s:s + 1], len(cols), axis=0)
        lnl = lf.part.batch_column_likelihoods(cols, Vs, case.root, weights=Ws,
                                               branch_k=case.branch_k if W is not None else None)
        out.append(normalise(lnl.reshape(L, D)))
    return np.stack(out)


@pytest.mark.parametrize("D,reversible", [(33, False), (48, True), (64, False)], ids=["33-nonrev", "48", "64-nonrev"])
def test_device_brute_force(D, reversible):
    for mix in (False, True):
        case, _ = sweep_support_case(D, reversible, mix)
        lf = new_lf(case)
        sup, _ = support_call(lf, case)
        want = device_brute(lf, case, range(3))
        lf.close()
        _, er = errors(sup[:3], want)
        print(f"[device brute D={D} mix={mix}] relative on entries >= {BIG:g}: {er:.2e}")
        assert er <= BRUTE_TOL


# ---------------------------------------------------------------------------------------------------------------------
# 7. bad input, chunks
# ---------------------------------------------------------------------------------------------------------------------
def test_nan_stays_in_its_set():
    for mix in (False, True):
        case, _ = sweep_support_case(61, True, mix)
        lf = new_lf(case)
        clean, site0 = support_call(lf, case)
        V = case.V.copy()
        V[3, 1, 0] = np.nan
        W = None
        if mix:
            W = case.W.copy()
            W[7, 2] = np.nan
        sup, site = support_call(lf, case, V=V, W=W)
        lf.close()
        bad = [3, 7] if mix else [3]
        for s in bad:
            assert np.isnan(site[s]) and np.isnan(sup[s]).any(), (mix, s)
        others = ~np.isin(np.arange(case.n), bad)
        assert np.array_equal(sup[others], clean[others]) and np.array_equal(site[others], site0[others])


@pytest.mark.parametrize("mix", [False, True], ids=["plain", "mix"])
def test_chunks_match_small_calls(mix):
    """More than 1024 sets (the chunk cap) in one call = the same sets in one-set and 100-set calls, bit for bit; the
    call runs exactly the launches of its two chunks; a repeated call is bit-identical."""
    w, _ = gc.load("mg94_8x60_c1")
    rng = np.random.default_rng(24 + mix)
    n = 1100
    branch_k, V, W, _ = meme_sets(w, 2, n, rng)
    if not mix:
        off = np.concatenate([[0], np.cumsum(branch_k)])
        V, W, branch_k = np.ascontiguousarray(V[:, off[:-1]]), None, None
    pats = rng.integers(0, w.S, n)
    lf = LF(w)
    part = lf.part

    def call(sl):
        return part.batch_leaf_support(pats[sl], V[sl], w.pi, weights=None if W is None else W[sl], branch_k=branch_k,
                                       want_site=True)
    l0 = part.launch_count
    sup, site = call(slice(0, n))
    l1 = part.launch_count
    a = call(slice(0, 1024))
    l2 = part.launch_count
    b = call(slice(1024, n))
    l3 = part.launch_count
    assert l1 - l0 == (l2 - l1) + (l3 - l2)
    assert np.all(np.isfinite(sup))
    assert np.array_equal(sup, np.concatenate([a[0], b[0]])) and np.array_equal(site, np.concatenate([a[1], b[1]]))
    for s0 in range(0, n, 100):
        p = call(slice(s0, s0 + 100))
        assert np.array_equal(p[0], sup[s0:s0 + 100]) and np.array_equal(p[1], site[s0:s0 + 100])
    for s in (0, 1023, 1024, n - 1):
        assert np.array_equal(call(slice(s, s + 1))[0][0], sup[s])
    again = call(slice(0, n))
    lf.close()
    assert np.array_equal(again[0], sup) and np.array_equal(again[1], site)


# ---------------------------------------------------------------------------------------------------------------------
# 8. non-interference, refusals
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("flags", [engine.FLAG_FORCE_FP64, engine.FLAG_DEFAULT])
def test_no_interference(flags):
    w, _ = gc.load("mg94_30x100_c4_ambig")
    rng = np.random.default_rng(25)
    lf = LF(w, flags)
    part = lf.part
    lf.set_all_matrices()
    before = lf.compute()
    part.branch_cache_build(5, w.pi)
    bc0 = part.branch_cache_evaluate(w.class_weights)
    branch_k, V, W, _ = meme_sets(w, 3, 40, rng)
    pats = rng.choice(w.S, 40)
    a = part.batch_leaf_support(pats, V, w.pi, weights=W, branch_k=branch_k, want_site=True)
    assert part.branch_cache_evaluate(w.class_weights) == bc0
    # the batch workspace handed to and from the other batch entry points, with other shapes
    rows = part.batch_branch_component_likelihoods(pats, V, W, w.pi, branch_k=branch_k)
    off = np.concatenate([[0], np.cumsum(branch_k)])
    Vp = np.ascontiguousarray(V[:, off[:-1]])
    plain = part.batch_site_likelihoods(pats, Vp, w.pi)
    b = part.batch_leaf_support(pats, V, w.pi, weights=W, branch_k=branch_k, want_site=True)
    c = part.batch_leaf_support(pats, Vp, w.pi, want_site=True)
    part.batch_site_simulate(Vp[:4], w.pi, 3)
    assert np.array_equal(part.batch_site_likelihoods(pats, Vp, w.pi), plain)
    assert np.array_equal(part.batch_branch_component_likelihoods(pats, V, W, w.pi, branch_k=branch_k)[1], rows[1])
    d = part.batch_leaf_support(pats, V, w.pi, weights=W, branch_k=branch_k, want_site=True)
    assert part.branch_cache_evaluate(w.class_weights) == bc0
    assert lf.compute() == before
    lf.close()
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and np.array_equal(a[0], d[0])
    assert np.array_equal(c[1], plain) and np.all(np.isfinite(c[0]))


def _raw(part, pats, K, branch_k, V, W, root, site, sup):
    po, ppo = _i(pats)
    pbk = None if branch_k is None else _i(branch_k)[1]
    pv = None if V is None else _d(V)[1]
    pw = None if W is None else _d(W)[1]
    ppi = None if root is None else _d(root)[1]
    ps = None if site is None else site.ctypes.data_as(_dp)
    pr = None if sup is None else sup.ctypes.data_as(_dp)
    return part._lib.hb2_batch_leaf_support(part._h, 0, len(po), ppo, int(K), pbk, pv, pw, None, ppi, ps, pr)


def test_refusals_leave_partition_usable():
    w, _ = gc.load("mg94_8x60_c1")
    rng = np.random.default_rng(26)
    branch_k, V, W, _ = meme_sets(w, 2, 8, rng)
    off = np.concatenate([[0], np.cumsum(branch_k)])
    Vp = np.ascontiguousarray(V[:, off[:-1]])
    pats = rng.choice(w.S, 8, replace=False)
    L, D = w.tree.n_leaves, w.D
    lf = LF(w)
    lf.set_all_matrices()
    lnl = lf.compute()
    good = lf.part.batch_leaf_support(pats, V, w.pi, weights=W, branch_k=branch_k, want_site=True)
    good_p = lf.part.batch_leaf_support(pats, Vp, w.pi, want_site=True)
    bad_k, bad_pat = branch_k.copy(), pats.copy()
    bad_k[0] = 3
    bad_pat[2] = w.S
    cases = [((pats, 0, branch_k, V, W, w.pi), "K=0 outside 1..4"), ((pats, 5, branch_k, V, W, w.pi), "K=5 outside 1..4"),
             ((pats, 2, bad_k, V, W, w.pi), r"branchK\[0\]=3 outside 1..2"),
             ((pats, 2, None, Vp, None, w.pi), "K=2 and branchK need weights"),
             ((pats, 1, branch_k, Vp, None, w.pi), "K=1 and branchK need weights"),
             ((pats, 2, branch_k, None, W, w.pi), "null argument"), ((pats, 2, branch_k, V, W, None), "null argument"),
             ((pats, 1, None, None, None, w.pi), "null argument"),
             ((bad_pat, 2, branch_k, V, W, w.pi), rf"patternOf\[2\]={w.S} out of range"),
             ((bad_pat, 1, None, Vp, None, w.pi), rf"patternOf\[2\]={w.S} out of range")]
    for args, msg in cases:
        site, sup = np.full(8, 7.0), np.full((8, L, D), 7.0)
        assert _raw(lf.part, *args, site, sup) != 0
        assert re.search(msg, lf.part._lib.hb2_last_error().decode()), lf.part._lib.hb2_last_error()
        assert np.all(site == 7.0) and np.all(sup == 7.0)
    for args in ((pats, 2, branch_k, V, W, w.pi), (pats, 1, None, Vp, None, w.pi)):
        site = np.full(8, 7.0)
        assert _raw(lf.part, *args, site, None) != 0
        assert "support must not be null" in lf.part._lib.hb2_last_error().decode()
        assert np.all(site == 7.0)
    # siteLnL is nullable
    sup = np.empty((8, L, D))
    _check(_raw(lf.part, pats, 2, branch_k, V, W, w.pi, None, sup))
    assert np.array_equal(sup, good[0])
    _check(_raw(lf.part, pats, 1, None, Vp, None, w.pi, None, sup))
    assert np.array_equal(sup, good_p[0])
    # nSets == 0 does nothing
    _check(_raw(lf.part, pats[:0], 2, branch_k, V[:0], W[:0], w.pi, np.empty(0), np.empty((0, L, D))))
    again = lf.part.batch_leaf_support(pats, V, w.pi, weights=W, branch_k=branch_k, want_site=True)
    assert np.array_equal(again[0], good[0]) and np.array_equal(again[1], good[1])
    assert lf.compute() == lnl
    lf.close()
    # 20 states: refused like the other batch entry points, and the partition still evaluates
    w20 = tree_workload(flat_tree(star(5)), 20, 40)
    lf = LikelihoodFunction(w20, flags=engine.FLAG_FORCE_FP64)
    lf.set_all_matrices()
    lnl = lf.compute()
    nb = w20.tree.n_branches
    sup = np.full((1, 5, 20), 7.0)
    assert _raw(lf.part, [0], 1, None, np.zeros((1, nb, 4)), None, w20.pi, np.empty(1), sup) != 0
    assert "33..64-state" in lf.part._lib.hb2_last_error().decode()
    assert np.all(sup == 7.0)
    assert lf.compute() == lnl
    lf.close()
