"""GPU suite (pytest -m gpu): the four batch entry points (hb2_batch_site_likelihoods, hb2_batch_site_mixture_likelihoods,
hb2_batch_column_likelihoods, hb2_batch_site_simulate) and their one host body at the shapes where the batch kernels branch,
every per-set value held to tests/batch_reference.py (long-double pruning; long-double exponentials where they are few,
the oracle's fp64 exponentials on the large trees):

  1. every state count 33..64 where the kernels change behaviour, with ambiguity rows, plain (FEL-shaped) and K = 4
     mixture (MEME-shaped) sets, a non-reversible template; fp64 and default partitions bit-identical;
  2. every tree shape of tests/test_gpu_shapes.py, including a 400-leaf star whose product leaves the double range;
  3. shared-powers group layouts: no hint, tested / background, 8 groups, groups of 3 and 4 rows, a wrong hint;
  4. column identities: probabilities of all D^3 columns of a 3-leaf star sum to 1; an ambiguity code is the sum over
     the states it allows;
  5. simulation draw by draw, on a 700-leaf caterpillar (internal states in global memory), across column launches, and
     against the scorer by a chi-square test;
  6. memory-derived chunks on the caterpillar: every result of a many-set call equals one-set calls bit for bit.

Unless a test says otherwise, sets use non-uniform root vectors and are checked with patterns and with columns."""
import dataclasses
import math

import numpy as np
import pytest
import scipy.stats

from hyphy_b200 import synth, LikelihoodFunction, engine
from oracle import port
from tests import batch_reference as br
from tests import simulate_reference as sim_ref
from tests import site_bootstrap_reference as sbr
from tests.test_gpu_shapes import TREES, flat_tree, inject_ambiguity, star

pytestmark = pytest.mark.gpu

# |got - ref| <= TOL[case] * |ref| per set: ten times the largest error measured on one H100 80GB HBM3 (700 W), rounded
# up to a power of ten (sweep 7.3e-16, shapes 1.8e-14 on the 400-leaf star and 7.6e-16 elsewhere, groups 1.9e-16,
# chunks 4.1e-16; DESIGN.md §2)
TOL = {"sweep": 1e-14, "shapes": 1e-12, "groups": 1e-14, "chunks": 1e-14}
HINT_TOL = 1e-13                    # a branch-group layout against the call without a hint
SUM_TOL = 1e-12                     # sum over all columns of exp(lnL) - 1
AMB_TOL = 1e-13                     # ambiguity marginalisation, relative

LENGTHS = np.array([0.02, 0.08, 0.2, 0.5, 1.2])          # branch lengths are drawn from these: few distinct matrices
LONG_LENGTHS = np.array([1.5, 3.0, 6.0])                  # 400-leaf star: every leaf costs several bits
SWEEP_TREE = [[0, [0, 0]], [0, 0, 0], 0, [0, 0]]          # 9 leaves, a 4-child root, a 3-child node
SWEEP = [(33, True), (40, True), (47, True), (48, True), (49, True), (61, True), (63, True), (64, True), (48, False)]
SIM_CHUNK, SIM_THREADS, SIM_SMEM_MAX = 1 << 18, 128, 48 << 10   # hb2_engine.cu
EXPM_POW_TERMS = 25                                              # hb2_kernels_fp64.cuh


@pytest.fixture(scope="module", autouse=True)
def _need_gpu(engine_lib):
    assert engine.device_count() > 0, "GPU tests need a CUDA device (no fallback exists)"


# ---------------------------------------------------------------------------------------------------------------------
# workloads
# ---------------------------------------------------------------------------------------------------------------------
@dataclasses.dataclass
class Case:
    """Sets on one partition: set s uses model mid[s] (its rows V[s], weights W[s]), pattern pats[s], column cols[s]."""
    tmpl: br.Template
    w: synth.Workload               # the partition: tree, patterns, ambiguity rows
    root: np.ndarray
    branch_k: np.ndarray            # [B]; ones for plain sets
    tested: np.ndarray              # [B] bool
    V: np.ndarray                   # [n, R, nF]
    W: np.ndarray | None            # [n, R]; None for plain sets
    mid: np.ndarray                 # [n]
    pats: np.ndarray                # [n]
    cols: np.ndarray                # [n, L]

    @property
    def mix(self):
        return self.W is not None

    @property
    def n(self):
        return len(self.V)


def make_tree(spec, seed, lengths=LENGTHS):
    tree = flat_tree(spec, seed=seed)
    tree.t = np.random.default_rng(seed).choice(lengths, len(tree.t))
    tree.t[-1] = 0.0
    return tree


def partition(tmpl, tree, n_sites, seed, amb_frac=0.0):
    """Patterns simulated on `tree` under the template at alpha = beta = 1; ambiguity rows injected on a fraction."""
    rng = np.random.default_rng(seed)
    D = tmpl.D
    pi0 = tmpl.cf if tmpl.cf is not None else np.full(D, 1.0 / D)
    Ps = [[np.maximum(synth._expm_np(br.dense(tmpl, br.row_values(tmpl, tree.t[b], 1.0, 1.0))), 0.0) for b in range(tree.n_branches)]]
    Ps = [[P / P.sum(axis=1, keepdims=True) for P in Ps[0]]]
    states = synth._simulate(tree, Ps, pi0, np.zeros(n_sites, dtype=np.int64), rng)
    ls, freq, s2p = synth.compress(states)
    w = synth.Workload(f"batch{tree.n_leaves}_D{D}", tree, D, pi0, [br.dense(tmpl, tmpl.base)], np.array([1.0]), ls,
                       np.zeros((0, D)), freq, s2p, None, {"kind": "generic"})
    if amb_frac:
        inject_ambiguity(w, rng, amb_frac)
    return w


def models(n, K, seed):
    rng = np.random.default_rng(seed)
    return [dict(alpha=rng.uniform(0.3, 2.0), beta_bg=rng.uniform(0.1, 3.0), betas=np.sort(rng.uniform(0.0, 6.0, K)),
                 wk=rng.dirichlet(np.ones(K))) for _ in range(n)]


def model_rows(tmpl, tree, branch_k, tested, m, mix):
    """(rows [R, nF], weights [R] | None) of one set model.  A branch of m >= 2 components (or a tested one) mixes
    betas[0..m-1] with weights wk[0..m-1] renormalised to sum 1; an untested branch is one row at beta_bg, weight 1."""
    V, W = [], []
    for b, k in enumerate(branch_k):
        t = tree.t[b]
        if not mix:
            V.append(br.row_values(tmpl, t, m["alpha"], m["betas"][0] if tested[b] else m["beta_bg"]))
            continue
        if k == 1 and not tested[b]:
            V.append(br.row_values(tmpl, t, m["alpha"], m["beta_bg"]))
            W.append(1.0)
            continue
        wk = m["wk"][:k] / m["wk"][:k].sum()
        for c in range(k):
            V.append(br.row_values(tmpl, t, m["alpha"], m["betas"][c]))
            W.append(wk[c])
    return np.array(V), (np.array(W) if mix else None)


def make_case(tmpl, w, n_sets, mix, K=4, branch_k=None, tested=None, n_models=2, seed=0, amb_cols=0.15):
    rng = np.random.default_rng(seed + 17)
    B = w.tree.n_branches
    if branch_k is None:
        branch_k = (np.arange(B) % K + 1) if mix else np.ones(B, np.int64)
    branch_k = np.asarray(branch_k, np.int64)
    if tested is None:
        tested = branch_k > 1 if mix else (np.arange(B) % 3 == 0)
    ms = models(n_models, K, seed)
    rows = [model_rows(tmpl, w.tree, branch_k, tested, m, mix) for m in ms]
    mid = np.arange(n_sets) % n_models
    V = np.stack([rows[i][0] for i in mid])
    W = np.stack([rows[i][1] for i in mid]) if mix else None
    if len(w.ambig):                                                        # patterns with ambiguity codes first
        amb = np.nonzero((w.leaf_states < 0).any(axis=0))[0]
        pats = np.concatenate([amb[:n_sets // 2], rng.integers(0, w.S, n_sets - min(len(amb), n_sets // 2))])
    else:
        pats = rng.integers(0, w.S, n_sets)
    cols = np.ascontiguousarray(w.leaf_states[:, rng.integers(0, w.S, n_sets)].T)
    if len(w.ambig) and amb_cols:
        hit = rng.random(cols.shape) < amb_cols
        cols[hit] = -(rng.integers(0, len(w.ambig), hit.sum()) + 1)
        cols[0, 0] = -1                                                     # the all-ones row
    root = np.random.default_rng(seed + 5).dirichlet(np.full(w.D, 2.0))
    return Case(tmpl, w, root, branch_k, np.asarray(tested, bool), V, W, mid, pats, cols)


def reference(case, expm, what, mutate=(), sets=None):
    """Long-double log-likelihoods of the sets (all, or `sets`) of `what` = "patterns" | "columns"."""
    Pm = {}
    out = []
    for s in (range(case.n) if sets is None else sets):
        if case.mid[s] not in Pm:
            Pm[case.mid[s]] = br.set_P(expm, case.V[s], None if case.W is None else case.W[s], case.branch_k, mutate)
        col = case.w.leaf_states[:, case.pats[s]] if what == "patterns" else case.cols[s]
        out.append(br.prune_ld(case.w.tree, Pm[case.mid[s]], col[None], case.w.ambig, case.root, mutate)[0])
    return np.array(out)


def expm_for(case):
    """Long-double exponentials where a case has few distinct rows, the oracle's fp64 ones on large trees."""
    return br.ExpmCache(case.tmpl, br.expm_ld if case.w.tree.n_branches < 100 else (lambda A: port.expm(A, False)))


def rel_err(got, ref):
    ref = np.asarray(ref, dtype=br.LD)
    return np.asarray(np.abs(np.asarray(got, dtype=br.LD) - ref) / np.abs(ref), dtype=np.float64)


# ---------------------------------------------------------------------------------------------------------------------
# engine calls
# ---------------------------------------------------------------------------------------------------------------------
def new_lf(case, flags=engine.FLAG_FORCE_FP64):
    lf = LikelihoodFunction(case.w, flags=flags)
    t = case.tmpl
    lf.part.set_rate_template(t.ei, t.ef, t.nF, t.cf)
    return lf


def run(lf, case, what, bg=None, V=None, W=None, pats=None, cols=None):
    V = case.V if V is None else V
    W = case.W if W is None else W
    bk = case.branch_k if case.mix else None
    if what == "patterns":
        pats = case.pats if pats is None else pats
        if not case.mix:
            return lf.part.batch_site_likelihoods(pats, V, case.root, branch_group=bg)
        return lf.part.batch_site_mixture_likelihoods(pats, V, W, case.root, branch_k=bk, branch_group=bg)
    cols = case.cols if cols is None else cols
    return lf.part.batch_column_likelihoods(cols, V, case.root, weights=W, branch_k=bk, branch_group=bg)


def check(case, got, ref, tol, label):
    err = rel_err(got, ref)
    assert np.all(np.isfinite(got)) and np.all(np.isfinite(np.asarray(ref, dtype=np.float64))), label
    print(f"[{label}] max |got - ref| / |ref| = {err.max():.2e} over {len(err)} sets")
    assert err.max() <= tol, (label, err.max(), int(err.argmax()))
    return err.max()


# ---------------------------------------------------------------------------------------------------------------------
# 1. state counts
# ---------------------------------------------------------------------------------------------------------------------
def sweep_case(D, reversible, mix, n_sets=12):
    tmpl = br.compact_template(D, reversible, seed=1)
    w = partition(tmpl, make_tree(SWEEP_TREE, seed=D), 120, seed=D, amb_frac=0.15)
    return make_case(tmpl, w, n_sets, mix, seed=D + (0 if reversible else 7))


@pytest.mark.parametrize("D,reversible", SWEEP, ids=[f"{d}{'' if r else '-nonrev'}" for d, r in SWEEP])
def test_state_sweep(D, reversible):
    for mix in (False, True):
        case = sweep_case(D, reversible, mix)
        if mix:
            assert set(case.branch_k) == {1, 2, 3, 4}
        expm = br.ExpmCache(case.tmpl, br.expm_ld)
        out = {}
        for flags in (engine.FLAG_FORCE_FP64, engine.FLAG_DEFAULT):
            lf = new_lf(case, flags)
            out[flags] = {what: run(lf, case, what) for what in ("patterns", "columns")}
            lf.close()
        for what in ("patterns", "columns"):
            got = out[engine.FLAG_FORCE_FP64][what]
            assert np.array_equal(got, out[engine.FLAG_DEFAULT][what]), what      # the batch path is fp64 under both
            src = case.w.leaf_states[:, case.pats].T if what == "patterns" else case.cols
            assert (src < 0).any() and (src == -1).any()
            check(case, got, reference(case, expm, what), TOL["sweep"], f"sweep D={D} rev={reversible} mix={mix} {what}")


# ---------------------------------------------------------------------------------------------------------------------
# 2. tree shapes
# ---------------------------------------------------------------------------------------------------------------------
SHAPES = [(s, D) for s in TREES for D in (61, 48)]


def shape_case(shape, D, mix, n_sets=6):
    tmpl = br.compact_template(D, True, seed=2)
    lengths = LONG_LENGTHS if shape == "star400" else LENGTHS
    w = partition(tmpl, make_tree(TREES[shape], seed=len(shape) + D, lengths=lengths), 60, seed=D + len(shape))
    return make_case(tmpl, w, n_sets, mix, seed=len(shape) + D)


@pytest.mark.parametrize("shape,D", SHAPES, ids=[f"{s}-{d}" for s, d in SHAPES])
def test_tree_shapes(shape, D):
    for mix in (False, True):
        case = shape_case(shape, D, mix)
        expm = expm_for(case)
        lf = new_lf(case)
        for what in ("patterns", "columns"):
            ref = reference(case, expm, what)
            if shape == "star400":                                          # the product leaves the double range
                assert np.all(np.asarray(ref, dtype=np.float64) < -1022 * math.log(2.0))
            check(case, run(lf, case, what), ref, TOL["shapes"], f"shape {shape} D={D} mix={mix} {what}")
        lf.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3. shared-powers group layouts
# ---------------------------------------------------------------------------------------------------------------------
def group_case(mix):
    """24 taxa, 61 states: 11 tested branches of K = 4 (3 in group 1, 4 in group 2, 2 with 3 background branches in
    group 3: components not proportional), the others background."""
    tmpl = br.compact_template(61, True, seed=3)
    tree = make_tree(_binary_spec(24, 3), seed=3)
    w = partition(tmpl, tree, 80, seed=3, amb_frac=0.05)
    B = tree.n_branches
    tested = np.zeros(B, bool)
    tested[np.random.default_rng(4).choice(B, 11, replace=False)] = True
    branch_k = np.where(tested, 4, 1) if mix else np.ones(B, np.int64)
    return make_case(tmpl, w, 10, mix, branch_k=branch_k, tested=tested, seed=3)


def _binary_spec(n, seed):
    """A random binary nested spec with a trifurcating root (n leaves)."""
    rng = np.random.default_rng(seed)
    nodes = [0] * n
    while len(nodes) > 3:
        i, j = sorted(rng.choice(len(nodes), 2, replace=False))
        b = nodes.pop(j)
        a = nodes.pop(i)
        nodes.append([a, b])
    return nodes


def layouts(case):
    B = case.w.tree.n_branches
    t = np.nonzero(case.tested)[0]
    designed = np.zeros(B, np.int64)
    designed[t[:3]], designed[t[3:7]], designed[t[7:9]] = 1, 2, 3
    designed[np.nonzero(~case.tested)[0][:3]] = 3
    designed[t[9:]] = 4
    return {"none": None, "tested": case.tested.astype(np.int64), "eight": np.arange(B, dtype=np.int64) % 8,
            "designed": designed}


def test_group_layouts():
    for mix in (False, True):
        case = group_case(mix)
        lay = layouts(case)
        d = lay["designed"]
        assert [int((d[case.tested] == g).sum()) for g in (1, 2)] == [3, 4]       # component groups of 3 and 4 rows
        assert (case.tested[d == 3]).any() and (~case.tested[d == 3]).any()      # a group of non-proportional rows
        assert len(set(lay["eight"])) == 8
        expm = br.ExpmCache(case.tmpl, br.expm_ld)
        lf = new_lf(case)
        for what in ("patterns", "columns"):
            ref = reference(case, expm, what)
            base = run(lf, case, what)
            for name, bg in lay.items():
                got = run(lf, case, what, bg=bg)
                check(case, got, ref, TOL["groups"], f"groups {name} mix={mix} {what}")
                assert np.all(rel_err(got, base) <= HINT_TOL), (name, what)
        lf.close()


def test_workspace_resize():
    """Calls on one partition whose chunks need more groups per set than the last call's (no hint, then 8 groups) re-size
    the batch workspace; each result, and a simulation after them, is bit-identical to the call on a fresh partition."""
    for mix in (False, True):
        case = group_case(mix)
        lay = layouts(case)
        calls = [(what, name) for name in ("none", "eight", "none", "tested") for what in ("patterns", "columns")]
        lf = new_lf(case)
        got = [run(lf, case, what, bg=lay[name]) for what, name in calls]
        sim = simulate(lf, case, 3, seed=11)
        lf.close()
        for (what, name), g in zip(calls, got):
            fresh = new_lf(case)
            assert np.array_equal(g, run(fresh, case, what, bg=lay[name])), (mix, what, name)
            fresh.close()
        fresh = new_lf(case)
        ref = simulate(fresh, case, 3, seed=11)
        fresh.close()
        assert np.array_equal(sim[0], ref[0]) and np.array_equal(sim[1], ref[1]), mix


# ---------------------------------------------------------------------------------------------------------------------
# 4. column identities
# ---------------------------------------------------------------------------------------------------------------------
def all_columns(D):
    return np.stack(np.unravel_index(np.arange(D ** 3), (D, D, D)), axis=1).astype(np.int64)


def star3_case(D, mix, seed=0):
    tmpl = br.compact_template(D, True, seed=4)
    w = partition(tmpl, make_tree(star(3), seed=seed + D), 20, seed=D)
    return make_case(tmpl, w, 1, mix, branch_k=np.full(3, 4) if mix else None, tested=np.ones(3, bool), seed=seed + D)


def column_lnl(lf, case, cols, per_call=32768):
    out = []
    for c0 in range(0, len(cols), per_call):
        n = len(cols[c0:c0 + per_call])
        V = np.broadcast_to(case.V[0], (n,) + case.V.shape[1:])
        W = None if case.W is None else np.broadcast_to(case.W[0], (n,) + case.W.shape[1:])
        out.append(run(lf, case, "columns", V=V, W=W, cols=cols[c0:c0 + per_call]))
    return np.concatenate(out)


@pytest.mark.parametrize("D", [33, 64])
def test_columns_sum_to_one(D):
    """Every column of a 3-leaf star is scored once: D = 64 runs 262 144 sets, 256 chunks of 1024."""
    cols = all_columns(D)
    for mix in (False, True):
        case = star3_case(D, mix)
        if mix:
            assert np.allclose(case.W[0].reshape(3, 4).sum(axis=1), 1.0)
        lf = new_lf(case)
        lnl = column_lnl(lf, case, cols)
        lf.close()
        assert np.all(np.isfinite(lnl))
        total = math.fsum(np.exp(lnl))
        print(f"[sum D={D} mix={mix}] |sum exp(lnL) - 1| = {abs(total - 1):.2e} over {len(cols)} columns")
        assert abs(total - 1.0) <= SUM_TOL


def test_ambiguity_marginalisation():
    """L(leaf l = row r) = sum over the states j that r allows of L(leaf l = j), for every row on every leaf."""
    tmpl = br.compact_template(47, True, seed=5)
    tree = make_tree([[0, 0], [0, [0, 0]], 0], seed=5)
    w = partition(tmpl, tree, 40, seed=5, amb_frac=0.1)
    L, D, nA = tree.n_leaves, w.D, len(w.ambig)
    base_cols = np.ascontiguousarray(w.leaf_states[:, :3].T.clip(0))
    for mix in (False, True):
        case = make_case(tmpl, w, 1, mix, seed=5)
        amb_cols, state_cols, owner = [], [], []
        for b in range(len(base_cols)):
            for leaf in range(L):
                for r in range(nA):
                    c = base_cols[b].copy()
                    c[leaf] = -(r + 1)
                    amb_cols.append(c)
                for j in range(D):
                    c = base_cols[b].copy()
                    c[leaf] = j
                    state_cols.append(c)
                owner.append((b, leaf))
        amb_cols, state_cols = np.array(amb_cols), np.array(state_cols)
        lf = new_lf(case)
        la = column_lnl(lf, case, amb_cols).reshape(-1, nA)
        ls = np.exp(column_lnl(lf, case, state_cols).reshape(-1, D))
        lf.close()
        want = np.log(ls @ w.ambig.T)
        err = np.abs(la - want)                                             # |ln(L_r / sum_j L_j)|: relative error of L
        print(f"[ambiguity mix={mix}] max relative error {err.max():.2e} over {la.size} columns")
        assert np.all(err <= AMB_TOL), err.max()


# ---------------------------------------------------------------------------------------------------------------------
# 5. simulation
# ---------------------------------------------------------------------------------------------------------------------
def simulate(lf, case, n_reps, seed, first_set=0, first_rep=0, want_nodes=True, V=None, W=None):
    V = case.V if V is None else V
    W = case.W if W is None else W
    return lf.part.batch_site_simulate(V, case.root, n_reps, weights=W, branch_k=case.branch_k if case.mix else None,
                                       seed=seed, first_set=first_set, first_rep=first_rep, want_nodes=want_nodes)


def check_draws(case, leaf, nodes, P_sets, seed, first_set, first_rep):
    """Every state given its parent's engine state is the reference draw from the fp64 matrix row on the stated uniform;
    a draw whose u*T lies within 1e-11*T of a prefix boundary may differ (the matrices agree to ~1e-13).  Returns their
    count."""
    tree = case.w.tree
    L, I, D = tree.n_leaves, tree.n_internal, case.w.D
    fp = tree.flat_parents
    reps = leaf.shape[1]
    g = np.arange(first_rep, first_rep + reps, dtype=np.uint64)
    rc, rl = sim_ref.prefix(case.root)
    near = 0
    for s in range(len(leaf)):
        t = np.uint64(first_set + s)
        state = np.concatenate([leaf[s], nodes[s]], axis=1).T
        u = sbr.uniforms(g, L + I - 1, t, seed)
        assert np.array_equal(state[-1], sim_ref.draw(np.broadcast_to(rc, (reps, D)), np.full(reps, rl), u))
        cdf, last = sim_ref.prefix(P_sets[s])
        for node in range(L + I - 1):
            par = state[L + fp[node]]
            u = sbr.uniforms(g, node, t, seed)
            c = cdf[node, par]
            want = sim_ref.draw(c, last[node, par], u)
            bad = np.nonzero(state[node] != want)[0]
            if len(bad):
                T = c[bad, -1]
                gap = np.abs(c[bad] - (u[bad] * T)[:, None]).min(axis=1)
                assert np.all(gap <= 1e-11 * T), (s, node, bad, state[node][bad], want[bad])
                near += len(bad)
    return near


def fp64_P(case, expm, sets):
    return np.stack([br.set_P(expm, case.V[s], None if case.W is None else case.W[s], case.branch_k).astype(np.float64)
                     for s in sets])


@pytest.mark.parametrize("D", [33, 47, 48, 64])
def test_simulation_draws(D):
    near = 0
    for mix in (False, True):
        case = sweep_case(D, True, mix, n_sets=4)
        expm = br.ExpmCache(case.tmpl, br.expm_ld)
        lf = new_lf(case)
        seed, first_set, first_rep = 0xBA7C4 + D, 77, 12345
        leaf, nodes = simulate(lf, case, 400, seed, first_set, first_rep)
        lf.close()
        near += check_draws(case, leaf, nodes, fp64_P(case, expm, range(case.n)), seed, first_set, first_rep)
    print(f"[sim D={D}] draws within 1e-11*T of a boundary that differ: {near}")
    assert near <= 5


def test_simulation_global_state_path():
    """A 700-leaf caterpillar: I = 698 internal nodes need I * 128 bytes > 48 KB, so states live in global memory."""
    near = 0
    for mix in (False, True):
        case = shape_case("caterpillar700", 61, mix, n_sets=2)
        assert case.w.tree.n_internal * SIM_THREADS > SIM_SMEM_MAX
        lf = new_lf(case)
        leaf, nodes = simulate(lf, case, 150, seed=99, first_set=5)
        lf.close()
        assert nodes.shape == (2, 150, case.w.tree.n_internal)
        near += check_draws(case, leaf, nodes, fp64_P(case, expm_for(case), range(2)), 99, 5, 0)
    print(f"[sim caterpillar700] draws within 1e-11*T of a boundary that differ: {near}")
    assert near <= 5


def test_simulation_launch_boundaries():
    """3 sets x 300 000 replicates: four column launches of 2^18, set 1 starting inside the second; the same columns as
    calls split by replicate and by set."""
    case = sweep_case(33, True, True, n_sets=3)
    reps, seed = 300_000, 4242
    ncol = case.n * reps
    assert -(-ncol // SIM_CHUNK) == 4 and SIM_CHUNK < reps < 2 * SIM_CHUNK
    lf = new_lf(case)
    simulate(lf, case, 1, seed)                                      # buffers sized; launch counts compared below
    n0 = lf.part.launch_count
    simulate(lf, case, 1, seed, want_nodes=False)
    one = lf.part.launch_count - n0
    n0 = lf.part.launch_count
    whole = simulate(lf, case, reps, seed)
    assert lf.part.launch_count - n0 == one + 3                     # three more column launches than a one-column call
    by_rep = [simulate(lf, case, r1 - r0, seed, first_rep=r0) for r0, r1 in ((0, 1000), (1000, 262_144), (262_144, reps))]
    by_set = [simulate(lf, case, reps, seed, first_set=s, V=case.V[s:s + 1], W=case.W[s:s + 1]) for s in range(case.n)]
    lf.close()
    for k in range(2):
        assert np.array_equal(whole[k], np.concatenate([p[k] for p in by_rep], axis=1))
        assert np.array_equal(whole[k], np.concatenate([p[k] for p in by_set], axis=0))
    assert len(np.unique(whole[0][:, ::1000].reshape(-1, case.w.tree.n_leaves), axis=0)) > 500


def test_simulation_agrees_with_scoring():
    """2^21 columns of one 33-state set on a 3-leaf star against exp(lnL) of all 35 937 columns from the column entry
    point; cells with an expected count below 5 pooled."""
    D, n = 33, 1 << 21
    for mix in (False, True):
        case = star3_case(D, mix, seed=1)
        lf = new_lf(case)
        p = np.exp(column_lnl(lf, case, all_columns(D)))
        leaf, _ = simulate(lf, case, n, seed=2024 + mix, want_nodes=False)
        lf.close()
        idx = (leaf[0, :, 0] * D + leaf[0, :, 1]) * D + leaf[0, :, 2]
        obs = np.bincount(idx, minlength=D ** 3).astype(float)
        exp = p * n
        small = exp < 5
        o = np.append(obs[~small], obs[small].sum())
        e = np.append(exp[~small], exp[small].sum())
        stat = ((o - e) ** 2 / e).sum()
        pval = scipy.stats.chi2.sf(stat, len(o) - 1)
        print(f"[chi2 mix={mix}] {len(o)} cells, statistic {stat:.1f}, p = {pval:.3f}")
        assert pval > 1e-4


# ---------------------------------------------------------------------------------------------------------------------
# 6. memory-derived chunks
# ---------------------------------------------------------------------------------------------------------------------
def chunk_cap(case, sim, rows=False):
    """Sets per chunk as batch_shape computes them (hb2_engine.cu), with no branch-group hint; `rows`: for
    hb2_batch_branch_component_likelihoods, whose messages, outside vectors and rows add to a mixture set's bytes."""
    B, I, D, nF = case.w.tree.n_branches, case.w.tree.n_internal, case.w.D, case.tmpl.nF
    R = int(case.branch_k.sum()) if case.mix else B
    sim_bytes = B * D * (64 * 8 + 4) if sim else 0.0
    if not case.mix:
        cap = int(8.0e9 / (B * (4096 + 1024 + nF) * 8 + sim_bytes))
    else:
        gk = int(case.branch_k.max())
        per_set = R * (4096 + nF + 1) * 8 + gk * EXPM_POW_TERMS * 4096 * 8 + I * 64 * 8
        if rows:
            per_set += B * 2 * (64 * 8 + 4) + R * 8
        cap = int(8.0e9 / (per_set + sim_bytes))
    return min(max(1, cap), 1024)


def chunk_case(mix, n_sets):
    tmpl = br.compact_template(61, True, seed=6)
    w = partition(tmpl, make_tree(TREES["caterpillar700"], seed=6), 40, seed=6, amb_frac=0.02)
    B = w.tree.n_branches
    return make_case(tmpl, w, n_sets, mix, branch_k=np.full(B, 4) if mix else None, n_models=3, seed=6)


@pytest.mark.parametrize("mix,n_sets", [(False, 300), (True, 100)], ids=["plain", "k4"])
def test_memory_chunks(mix, n_sets):
    case = chunk_case(mix, n_sets)
    caps = {sim: chunk_cap(case, sim) for sim in (False, True)}
    assert all(n_sets > 2 * c for c in caps.values()), caps                   # three chunks or more, every entry point
    print(f"[chunks mix={mix}] {n_sets} sets, {caps[False]} per likelihood chunk, {caps[True]} per simulation chunk")
    lf = new_lf(case)
    whole = {what: run(lf, case, what) for what in ("patterns", "columns")}
    sim_whole = simulate(lf, case, 2, seed=31)
    for s in range(n_sets):
        V, W = case.V[s:s + 1], None if case.W is None else case.W[s:s + 1]
        for what in ("patterns", "columns"):
            one = run(lf, case, what, V=V, W=W, pats=case.pats[s:s + 1], cols=case.cols[s:s + 1])
            assert one[0] == whole[what][s], (what, s)
        leaf, nodes = simulate(lf, case, 2, seed=31, first_set=s, V=V, W=W)
        assert np.array_equal(leaf[0], sim_whole[0][s]) and np.array_equal(nodes[0], sim_whole[1][s]), s
    lf.close()
    expm = expm_for(case)
    for what in ("patterns", "columns"):
        sets = [0, caps[False], n_sets - 1]                                   # first set of the first, second and last chunk
        check(case, whole[what][sets], reference(case, expm, what, sets=sets), TOL["chunks"], f"chunks mix={mix} {what}")
