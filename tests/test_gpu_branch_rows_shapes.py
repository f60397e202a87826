"""GPU suite (pytest -m gpu): hb2_batch_branch_component_likelihoods (branch_rows_kernel and its host path) at the shapes
where they branch, on the workloads of tests/test_gpu_batch_shapes.py, every row held to tests/branch_rows_reference.py
(long-double brute force, MEME's own procedure, on small trees; the long-double outside pass on trees of 100 branches or
more):

  1. every state count 33..64 where the kernels change behaviour, reversible and not, with ambiguity rows and branchK
     taking 1..4 in one set; fp64 and default partitions bit-identical; one-component branches equal to the site;
  2. the caller's root vector: Dirichlet, uniform, and one with zeros in a third of the states;
  3. exact identities: a branch's rows do not depend on its own weights (zero or unnormalised) nor on its other
     components' formula values, bit for bit; an identity exponential next to finite components;
  4. every tree shape of tests/test_gpu_shapes.py at 48 states, including a 400-leaf star below 2^-1022;
  5. shared-powers group layouts;
  6. memory-derived chunks (the branch-rows term of the chunk rule) equal to one-set calls bit for bit;
  7. the batch workspace handed between branch-rows calls of other shapes and the other batch entry points;
  8. template 1 next to a different template 0, and new column frequencies;
  9. formula values past the exponential's range, or NaN: NaN for their set only.

Unless a test says otherwise every call uses the case's Dirichlet root vector (not the model's stationary vector), and
every call checks that siteLnL is hb2_batch_site_mixture_likelihoods' bit for bit and that every branch of a set with a
finite site mixes back to it: log sum_k w_k exp(row_{b,k} - site) = 0."""
import dataclasses
import functools
import itertools
import math

import numpy as np
import pytest

from hyphy_b200 import LikelihoodFunction, engine
from tests import batch_reference as br
from tests import branch_rows_reference as brr
from tests.test_gpu_batch_shapes import (SWEEP, HINT_TOL, chunk_cap, chunk_case, expm_for, group_case, layouts, make_case,
                                         new_lf, rel_err, run, shape_case, simulate, sweep_case)
from tests.test_gpu_branch_rows import mixture_identity, offsets
from tests.test_gpu_shapes import TREES

pytestmark = pytest.mark.gpu

# Ten times the largest error measured on one H100 80GB HBM3 (700 W), rounded up to a power of ten (DESIGN.md §2).
# |row - ref| <= TOL[case] * |ref| per row: sweep 9.3e-16 (the root, identity and template tests included), shapes 2.5e-15
# on the 400-leaf star and 5.6e-16 elsewhere, groups 1.6e-16, chunks 5.4e-16
TOL = {"sweep": 1e-14, "shapes": 1e-13, "groups": 1e-14, "chunks": 1e-14}
ID_TOL = 1e-11                      # |log sum_k w_k exp(row_{b,k} - site)|: 2.0e-13 (400-leaf star, 700-leaf caterpillar)
ONE_TOL = 1e-14                     # a one-component branch's row against the site, relative: 2.2e-16
SWEEP_ROWS = SWEEP + [(33, False), (64, False)]
IDENTITY = [(33, False), (48, True), (64, False)]


@pytest.fixture(scope="module", autouse=True)
def _need_gpu(engine_lib):
    assert engine.device_count() > 0, "GPU tests need a CUDA device (no fallback exists)"


# ---------------------------------------------------------------------------------------------------------------------
# calls and references
# ---------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def sweep_rows_case(D, reversible):
    """The K = 4 sweep workload of the batch-shapes file and its long-double exponentials (shared between tests: treat
    both as read-only)."""
    case = sweep_case(D, reversible, True)
    return case, br.ExpmCache(case.tmpl, br.expm_ld)


def branch_rows(lf, case, V=None, W=None, root=None, bg=None, template=0):
    V = case.V if V is None else V
    W = case.W if W is None else W
    root = case.root if root is None else root
    return lf.part.batch_branch_component_likelihoods(case.pats, V, W, root, branch_k=case.branch_k, branch_group=bg,
                                                      template=template)


def check_call(lf, case, site, rows, V=None, W=None, root=None, bg=None, template=0):
    """siteLnL = the mixture call's on the same arguments, bit for bit; every branch of a finite set mixes back to it."""
    V = case.V if V is None else V
    W = case.W if W is None else W
    root = case.root if root is None else root
    mixed = lf.part.batch_site_mixture_likelihoods(case.pats, V, W, root, branch_k=case.branch_k, branch_group=bg,
                                                   template=template)
    assert np.array_equal(site, mixed, equal_nan=True)
    ok = np.isfinite(site)
    if ok.any():
        err = float(np.abs(mixture_identity(case.branch_k, W[ok], site[ok], rows[ok])).max())
        assert err <= ID_TOL, err
        return err
    return 0.0


def rows_call(lf, case, **kw):
    site, rows = branch_rows(lf, case, **kw)
    err = check_call(lf, case, site, rows, **kw)
    print(f"  identity: max |log sum_k w_k exp(row - site)| = {err:.2e}")
    return site, rows


def ref_rows(case, expm, sets, V=None, W=None, root=None, outside=False):
    """Long-double rows [len(sets), R]: brute force, or the outside pass (`outside`)."""
    V = case.V if V is None else V
    W = case.W if W is None else W
    root = case.root if root is None else root
    fn = brr.outside_rows if outside else brr.brute_rows
    with np.errstate(divide="ignore"):
        return np.stack([fn(case.w.tree, expm, V[s], W[s], case.branch_k, case.w.leaf_states[:, case.pats[s]], case.w.ambig,
                            root) for s in sets])


def check_rows(got, ref, tol, label):
    """Finite exactly where the reference is, -inf where it is -inf, and within tol relative elsewhere."""
    ref64 = np.asarray(ref, dtype=np.float64)
    fin = np.isfinite(ref64)
    assert np.array_equal(np.isfinite(got), fin), label
    assert np.array_equal(got[~fin], ref64[~fin]), label
    err = rel_err(got[fin], ref[fin]) if fin.any() else np.zeros(1)
    print(f"[{label}] max |row - ref| / |ref| = {err.max():.2e} over {fin.sum()} rows ({(~fin).sum()} -inf)")
    assert err.max() <= tol, (label, err.max())
    return err.max()


def mixed_branch(case):
    """A branch of the most components, internal if one is (its outside vector feeds the rows below it)."""
    L, k = case.w.tree.n_leaves, case.branch_k
    cand = np.nonzero(k == k.max())[0]
    internal = cand[cand >= L]
    return int(internal[0] if len(internal) else cand[0])


# ---------------------------------------------------------------------------------------------------------------------
# 1. state counts
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D,reversible", SWEEP_ROWS, ids=[f"{d}{'' if r else '-nonrev'}" for d, r in SWEEP_ROWS])
def test_state_sweep(D, reversible):
    case, expm = sweep_rows_case(D, reversible)
    assert set(case.branch_k) == {1, 2, 3, 4}
    src = case.w.leaf_states[:, case.pats]
    assert (src < 0).any() and (src == -1).any()                            # ambiguity codes, the all-ones row among them
    out = {}
    for flags in (engine.FLAG_FORCE_FP64, engine.FLAG_DEFAULT):
        lf = new_lf(case, flags)
        out[flags] = rows_call(lf, case)
        lf.close()
    site, rows = out[engine.FLAG_FORCE_FP64]
    assert np.array_equal(site, out[engine.FLAG_DEFAULT][0]) and np.array_equal(rows, out[engine.FLAG_DEFAULT][1])
    check_rows(rows, ref_rows(case, expm, range(case.n)), TOL["sweep"], f"sweep D={D} rev={reversible}")
    one = offsets(case.branch_k)[:-1][case.branch_k == 1]
    err = np.abs(rows[:, one] - site[:, None]) / np.abs(site[:, None])
    print(f"  one-component rows against the site: {err.max():.2e}")
    assert err.max() <= ONE_TOL


# ---------------------------------------------------------------------------------------------------------------------
# 2. the caller's root vector
# ---------------------------------------------------------------------------------------------------------------------
def test_root_vectors():
    case, expm = sweep_rows_case(48, False)
    D = case.w.D
    rng = np.random.default_rng(48)
    sparse = np.zeros(D)
    keep = rng.permutation(D)[:D - D // 3]
    sparse[keep] = rng.dirichlet(np.full(len(keep), 2.0))
    roots = {"dirichlet": case.root, "uniform": np.full(D, 1.0 / D), "zeros": sparse}
    lf = new_lf(case)
    got = {}
    for name, root in roots.items():
        _, got[name] = rows_call(lf, case, root=root)
        check_rows(got[name], ref_rows(case, expm, range(case.n), root=root), TOL["sweep"], f"root {name}")
    lf.close()
    for a, b in itertools.combinations(roots, 2):
        shift = np.median(rel_err(got[a], got[b]))
        print(f"  rows under {a} and {b} roots: median relative difference {shift:.2e}")
        assert shift > 1e3 * TOL["sweep"], (a, b)


# ---------------------------------------------------------------------------------------------------------------------
# 3. exact identities
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D,reversible", IDENTITY, ids=[f"{d}{'' if r else '-nonrev'}" for d, r in IDENTITY])
def test_rows_ignore_own_weights(D, reversible):
    """Branch b's weights set to zeros, to a sum of 0.3 and to a sum of 3: b's rows do not move by one bit; the site and
    every other row do, and match the reference; the mixture identity holds with the unnormalised weights."""
    case, expm = sweep_rows_case(D, reversible)
    b = mixed_branch(case)
    off = offsets(case.branch_k)
    own = np.zeros(off[-1], bool)
    own[off[b]:off[b + 1]] = True
    rng = np.random.default_rng(D)
    lf = new_lf(case)
    site0, rows0 = rows_call(lf, case)
    for total in (0.0, 0.3, 3.0):
        W = case.W.copy()
        W[:, own] = total * rng.dirichlet(np.ones(own.sum()), case.n)
        site, rows = rows_call(lf, case, W=W)
        assert np.array_equal(rows[:, own], rows0[:, own]), total
        assert np.all(site != site0) and np.all(rows[:, ~own] != rows0[:, ~own]), total
        if total == 0.0:
            assert np.all(site == -np.inf) and np.all(rows[:, ~own] == -np.inf)
        check_rows(rows, ref_rows(case, expm, range(case.n), W=W), TOL["sweep"], f"weights D={D} sum={total}")
    lf.close()


@pytest.mark.parametrize("D,reversible", IDENTITY, ids=[f"{d}{'' if r else '-nonrev'}" for d, r in IDENTITY])
def test_rows_ignore_other_components(D, reversible):
    """Component r of branch b gets other formula values: b's other rows do not move by one bit, row r matches the
    reference.  b is alone in its branch group in both calls, so no shared-powers group holds r and another branch."""
    case, expm = sweep_rows_case(D, reversible)
    b = mixed_branch(case)
    off = offsets(case.branch_k)
    r = int(off[b] + 1)
    rest = [q for q in range(off[b], off[b + 1]) if q != r]
    bg = np.zeros(case.w.tree.n_branches, np.int64)
    bg[b] = 1
    lf = new_lf(case)
    _, rows0 = rows_call(lf, case, bg=bg)
    V = case.V.copy()
    V[:, r] *= 1.7
    _, rows = rows_call(lf, case, V=V, bg=bg)
    lf.close()
    assert np.array_equal(rows[:, rest], rows0[:, rest])
    assert np.all(rows[:, r] != rows0[:, r])
    check_rows(rows, ref_rows(case, expm, range(case.n), V=V), TOL["sweep"], f"components D={D}")


@pytest.mark.parametrize("D,reversible", IDENTITY, ids=[f"{d}{'' if r else '-nonrev'}" for d, r in IDENTITY])
def test_identity_component(D, reversible):
    """One row of zero formula values (its exponential is the identity) next to finite components."""
    case, expm = sweep_rows_case(D, reversible)
    b = mixed_branch(case)
    r = int(offsets(case.branch_k)[b] + 2)
    V = case.V.copy()
    V[:, r] = 0.0
    lf = new_lf(case)
    _, rows = rows_call(lf, case, V=V)
    lf.close()
    check_rows(rows, ref_rows(case, expm, range(case.n), V=V), TOL["sweep"], f"identity row D={D}")
    assert np.all(np.isfinite(np.delete(rows, r, axis=1)))


# ---------------------------------------------------------------------------------------------------------------------
# 4. tree shapes
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", list(TREES))
def test_tree_shapes(shape):
    case = shape_case(shape, 48, True)
    big = case.w.tree.n_branches >= 100                # brute force costs R prunings per set: the outside pass there
    expm = expm_for(case)
    lf = new_lf(case)
    _, rows = rows_call(lf, case)
    lf.close()
    sets = [0, 1] if big else range(case.n)
    ref = ref_rows(case, expm, sets, outside=big)
    if shape == "star400":                             # the product leaves the double range
        site = [brr.site_ld(case.w.tree, expm, case.V[s], case.W[s], case.branch_k, case.w.leaf_states[:, case.pats[s]],
                            case.w.ambig, case.root) for s in sets]
        assert np.all(np.asarray(site, dtype=np.float64) < -1022 * math.log(2.0))
    check_rows(rows[list(sets)], ref, TOL["shapes"], f"shape {shape} D=48")


# ---------------------------------------------------------------------------------------------------------------------
# 5. shared-powers group layouts
# ---------------------------------------------------------------------------------------------------------------------
def test_group_layouts():
    case = group_case(True)
    lay = layouts(case)
    expm = br.ExpmCache(case.tmpl, br.expm_ld)
    ref = ref_rows(case, expm, range(case.n))
    lf = new_lf(case)
    _, base = rows_call(lf, case)
    for name, bg in lay.items():
        _, got = rows_call(lf, case, bg=bg)
        check_rows(got, ref, TOL["groups"], f"groups {name}")
        assert np.all(rel_err(got, base) <= HINT_TOL), name
    lf.close()


# ---------------------------------------------------------------------------------------------------------------------
# 6. memory-derived chunks
# ---------------------------------------------------------------------------------------------------------------------
def test_memory_chunks():
    """100 sets of R = 5588 rows (K = 4 on the 700-leaf caterpillar): the chunk rule with the branch-rows term gives three
    or more chunks.  The call runs the launches of its chunks called separately, and every set equals a one-set call."""
    n = 100
    case = chunk_case(True, n)
    cap = chunk_cap(case, False, rows=True)
    assert n > 2 * cap and cap < 1024, cap
    print(f"[chunks] {n} sets of {case.V.shape[1]} rows, {cap} per branch-rows chunk")
    lf = new_lf(case)
    part = lf.part
    l0 = part.launch_count
    site, rows = branch_rows(lf, case)
    whole = part.launch_count - l0
    check_call(lf, case, site, rows)
    starts = list(range(0, n, cap))
    parts = 0
    for s0 in starts:
        sub = slice(s0, s0 + cap)
        l0 = part.launch_count
        part.batch_branch_component_likelihoods(case.pats[sub], case.V[sub], case.W[sub], case.root, branch_k=case.branch_k)
        parts += part.launch_count - l0
    assert whole == parts, (whole, parts)
    for s in range(n):
        one = dataclasses.replace(case, V=case.V[s:s + 1], W=case.W[s:s + 1], pats=case.pats[s:s + 1])
        s1, r1 = branch_rows(lf, one)
        check_call(lf, one, s1, r1)
        assert s1[0] == site[s] and np.array_equal(r1[0], rows[s]), s
    lf.close()
    sets = [0, starts[1], starts[-1]]                 # first set of the first, second and last chunk
    check_rows(rows[sets], ref_rows(case, expm_for(case), sets, outside=True), TOL["chunks"], "chunks")


# ---------------------------------------------------------------------------------------------------------------------
# 7. workspace hand-over
# ---------------------------------------------------------------------------------------------------------------------
def head(case, n):
    return dataclasses.replace(case, V=case.V[:n], W=case.W[:n], mid=case.mid[:n], pats=case.pats[:n], cols=case.cols[:n])


def test_workspace_handover():
    """One partition: branch rows (3 sets, R = 78), a mixture call (10 sets), branch rows (3 sets, R = 180 on K = 4
    everywhere), a column call, a simulation, the first call again.  The workspace is re-sized into and out of the
    branch-rows buffers, and the last calls reuse them; each result equals the call on a fresh partition bit for bit."""
    case = group_case(True)
    small = head(case, 3)
    B = case.w.tree.n_branches
    wide = make_case(case.tmpl, case.w, 3, True, branch_k=np.full(B, 4), tested=np.ones(B, bool), seed=8)
    assert wide.V.shape[1] > small.V.shape[1]
    calls = [("rows", small), ("mixture", case), ("rows", wide), ("columns", small), ("simulate", small), ("rows", small)]

    def call(lf, what, c):
        if what == "rows":
            return branch_rows(lf, c)
        if what == "simulate":
            return simulate(lf, c, 3, seed=11)
        return (run(lf, c, "patterns" if what == "mixture" else "columns"),)

    lf = new_lf(case)
    got = [call(lf, what, c) for what, c in calls]
    lf.close()
    for (what, c), g in zip(calls, got):
        fresh = new_lf(case)
        want = call(fresh, what, c)
        if what == "rows":
            check_call(fresh, c, *want)
        fresh.close()
        assert all(np.array_equal(a, b) for a, b in zip(g, want)), what


# ---------------------------------------------------------------------------------------------------------------------
# 8. template 1 and new column frequencies
# ---------------------------------------------------------------------------------------------------------------------
def two_templates(case, tmpl1):
    lf = LikelihoodFunction(case.w, flags=engine.FLAG_FORCE_FP64)
    other = br.compact_template(case.w.D, False, seed=9)    # other formulas, no column frequencies
    lf.part.set_rate_template_id(0, other.ei, other.ef, other.nF, other.cf)
    lf.part.set_rate_template_id(1, tmpl1.ei, tmpl1.ef, tmpl1.nF, tmpl1.cf)
    return lf


def test_template_one_and_frequencies():
    """Rows under template 1, with template 0 defined differently, equal those of a partition where it is template 0.
    New column frequencies for template 1: the next call matches the reference under them (no power table of the old
    frequencies survives), and equals a partition whose template 1 was defined with them."""
    case, expm = sweep_rows_case(48, True)
    lf = two_templates(case, case.tmpl)
    site1, rows1 = rows_call(lf, case, template=1)
    fresh = new_lf(case)
    site0, rows0 = rows_call(fresh, case)
    fresh.close()
    assert np.array_equal(site1, site0) and np.array_equal(rows1, rows0)
    t2 = dataclasses.replace(case.tmpl, cf=np.random.default_rng(49).dirichlet(np.full(case.w.D, 5.0)))
    lf.part.set_template_frequencies(1, t2.cf)
    site2, rows2 = rows_call(lf, case, template=1)
    lf.close()
    assert np.all(rows2 != rows1)
    case2 = dataclasses.replace(case, tmpl=t2)
    check_rows(rows2, ref_rows(case2, br.ExpmCache(t2, br.expm_ld), range(case.n)), TOL["sweep"], "template 1, new frequencies")
    fresh = two_templates(case, t2)
    site3, rows3 = rows_call(fresh, case, template=1)
    fresh.close()
    assert np.array_equal(site2, site3) and np.array_equal(rows2, rows3)


# ---------------------------------------------------------------------------------------------------------------------
# 9. formula values out of range or NaN
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bad", ["range", "nan"])
def test_bad_row_stays_in_its_set(bad):
    """Row r of branch b in set 5: values past the exponential's range (scaling shift > 900) or a NaN.  That set's site
    and row r are NaN; b's other rows, which never read b's matrix, keep every bit; every other set keeps every bit.
    b is alone in its branch group in both calls."""
    case, _ = sweep_rows_case(48, False)
    b = mixed_branch(case)
    off = offsets(case.branch_k)
    r = int(off[b] + 1)
    rest = [q for q in range(off[b], off[b + 1]) if q != r]
    bg = np.zeros(case.w.tree.n_branches, np.int64)
    bg[b] = 1
    s = 5
    V = case.V.copy()
    if bad == "range":
        V[s, r] *= 1e280
        M = np.abs(br.dense(case.tmpl, V[s, r]))
        assert min(M.sum(axis=0).max(), M.sum(axis=1).max()) > 0.975 * 2.0 ** 901
    else:
        V[s, r, 0] = np.nan
    lf = new_lf(case)
    site0, rows0 = rows_call(lf, case, bg=bg)
    site, rows = rows_call(lf, case, V=V, bg=bg)
    lf.close()
    assert np.isnan(site[s]) and np.isnan(rows[s, r])
    assert np.array_equal(rows[s, rest], rows0[s, rest])
    others = np.arange(case.n) != s
    assert np.array_equal(site[others], site0[others]) and np.array_equal(rows[others], rows0[others])
