"""GPU suite (pytest -m gpu): every padded state size, pattern-count edges, tree shapes and kernel variants against the oracle.

test_gpu_parity.py covers 61 codon states and 4 nucleotides on binary trees thoroughly; this module covers the rest:
  * a state-count sweep over both ends and the inside of every padding bucket (Dp = 4, 8, 16, 24, 32, 64): kernel
    selection, transition matrices at the norms where a scaled Taylor series is weakest, compiled hand-over, likelihoods,
    partial updates, forced states, branch cache, conditionals' read-back, impossible patterns and NaN;
  * pattern counts at the edges of a 128-pattern tile (S = 1, 2, 127, 129, 300);
  * star trees, internal polytomies, a bifurcating root, a caterpillar (every step a register hand-over), a leaf next to
    a deep subtree;
  * switches that choose between kernel shapes, which must not change the results;
  * star trees whose product over children underflows a double before the end of the node.
Tolerances are those of test_gpu_parity.py: fp64 kernels 1e-10 relative on lnL and 1e-8 per pattern, the tensor path
(33..64 states without HB2_FLAG_FORCE_FP64) 1e-7 and 1e-5."""
import numpy as np
import pytest
import scipy.linalg

from hyphy_b200 import synth, LikelihoodFunction, engine
from oracle import port
from tests import resident_reference as rr

pytestmark = pytest.mark.gpu

MODES = {"fp64": (engine.FLAG_FORCE_FP64, 1e-10, 1e-8),     # flags, lnL rtol, per-pattern atol
         "tc": (engine.FLAG_DEFAULT, 1e-7, 1e-5)}


@pytest.fixture(scope="module", autouse=True)
def _need_gpu(engine_lib):
    assert engine.device_count() > 0, "GPU tests need a CUDA device (no fallback exists)"


def LF(w, mode):
    return LikelihoodFunction(w, flags=MODES[mode][0])


def tol(w, mode):
    if mode == "tc" and w.D > 32:
        return MODES["tc"][1], MODES["tc"][2]
    return MODES["fp64"][1], MODES["fp64"][2]


def with_modes(Ds):
    """(D, mode) pairs: fp64 for every D; the tensor path only where it exists (33..64 states), so no case runs twice."""
    return [(D, "fp64") for D in Ds] + [(D, "tc") for D in Ds if D > 32]


def _site_lnl(sl, ss):
    return np.log(sl) - 64.0 * np.log(2.0) * ss


def pad_states(D):
    return next(p for p in (4, 8, 16, 24, 32, 64) if D <= p)


# ---------------------------------------------------------------------------------------------------------------------
# trees and workloads
# ---------------------------------------------------------------------------------------------------------------------
def flat_tree(spec, mean_t=0.2, seed=0):
    """synth.FlatTree from a nested children list: a leaf is 0, an internal node the list of its children, `spec` the
    root.  Leaves and internal nodes get post-order ids (leaves 0..L-1, internal nodes L..L+I-1, root last)."""
    obj, par = [spec], [-1]
    i = 0
    while i < len(obj):                                   # breadth-first: parents before children
        if isinstance(obj[i], list):
            assert len(obj[i]) >= 2, "an internal node needs two children or more"
            for c in obj[i]:
                obj.append(c)
                par.append(i)
        i += 1
    kids = [[] for _ in obj]
    for j in range(1, len(obj)):
        kids[par[j]].append(j)
    post, stack = [], [(0, 0)]
    while stack:                                          # iterative post-order (caterpillars are deep)
        n, ci = stack.pop()
        if ci < len(kids[n]):
            stack.append((n, ci + 1))
            stack.append((kids[n][ci], 0))
        else:
            post.append(n)
    leaves = [n for n in post if not kids[n]]
    internals = [n for n in post if kids[n]]
    L, I = len(leaves), len(internals)
    fid = {n: k for k, n in enumerate(leaves)}
    fid.update({n: L + k for k, n in enumerate(internals)})
    fp = np.full(L + I, -1, dtype=np.int64)
    for n in post:
        if par[n] >= 0:
            fp[fid[n]] = fid[par[n]] - L
    t = np.maximum(np.random.default_rng(seed).exponential(mean_t, L + I), 1e-4)
    t[L + I - 1] = 0.0
    names = [f"T{k + 1}" for k in range(L)] + [f"N{k + 1}" for k in range(I)]
    return synth.FlatTree(L, I, fp, names, t, "")


def star(n):
    return [0] * n


def polytomy(k):
    """Root (trifurcating) with a child of k children: leaves and cherries alternate under it."""
    return [[0 if i % 2 == 0 else [0, 0] for i in range(k)], [0, 0], 0]


def caterpillar(n):
    c = [0, 0]
    for _ in range(n - 4):
        c = [c, 0]
    return [c, 0, 0]


TREES = {
    "star3": star(3),
    "star40": star(40),
    "star400": star(400),
    "poly3": polytomy(3),
    "poly4": polytomy(4),
    "poly7": polytomy(7),
    "poly33": polytomy(33),
    "all_internal": [[[0, 0], [0, [0, 0]], [0, 0, 0]], 0, 0],        # a node whose three children are all internal
    "bifurcating_root": [[0, [0, 0]], [[0, 0], [0, 0, 0]]],
    "caterpillar700": caterpillar(700),
    "leaf_by_deep": [0, caterpillar(40)],                             # a leaf hanging off the root next to a deep subtree
}


def model(D, seed=0):
    """Random reversible D-state model (61 states: MG94xREV, with the codon meta of synth.codon_workload)."""
    if D == 61:
        return synth.mg94_rev_Q(0.5), synth.codon_frequencies(synth.DEFAULT_POSFREQ), {
            "kind": "codon", "theta": synth.DEFAULT_THETA.tolist(), "posfreq": synth.DEFAULT_POSFREQ.tolist(), "omegas": [0.5]}
    Q, pi = synth.gtr_like_Q(D, seed + D)
    return Q, pi, {"kind": "generic"}


def tree_workload(tree, D, n_sites, seed=0, n_patterns=None):
    """One rate class, data simulated on `tree`; the first n_patterns unique patterns if given."""
    rng = np.random.default_rng(seed + 7 * D + n_sites)
    Q, pi, meta = model(D, seed)
    nb = tree.n_branches
    Ps = [[synth._expm_np(Q * tree.t[b]) for b in range(nb)]]
    states = synth._simulate(tree, Ps, pi, np.zeros(n_sites, dtype=np.int64), rng)
    ls, freq, s2p = synth.compress(states)
    if n_patterns is not None:
        assert ls.shape[1] >= n_patterns
        ls, freq = ls[:, :n_patterns].copy(), freq[:n_patterns].copy()
        s2p = np.arange(n_patterns)
    return synth.Workload(f"tree{tree.n_leaves}_D{D}", tree, D, pi, [Q], np.array([1.0]), ls, np.zeros((0, D)), freq, s2p,
                          None, meta)


def inject_ambiguity(w, rng, frac=0.05):
    """Random 0/1 resolution rows, one of them all ones, on a fraction of the leaf cells."""
    amb = (rng.random((5, w.D)) < 0.3).astype(float)
    amb[np.arange(5), rng.integers(0, w.D, 5)] = 1.0
    amb[0] = 1.0
    ls = w.leaf_states.copy()
    hit = rng.random(ls.shape) < frac
    ls[hit] = -(rng.integers(0, 5, size=hit.sum()) + 1)
    ls[0, 0] = -1                                                     # the all-ones row is used at least once
    w.ambig, w.leaf_states = amb, ls


def sparse(w):
    """Codon models take the reference's sparse-storage scaling in the oracle's expm (as port.lnl does for 61 states)."""
    return w.meta.get("kind") == "codon"


def oracle_P(w, c=0, Qt=None):
    """The oracle's transition matrices of class c."""
    Qt = w.Qt() if Qt is None else Qt
    return np.stack([port.expm(q, sparse(w)) for q in Qt[c]])


def oracle_sites(w, P):
    sl, ss = port.prune(w, P)
    site = _site_lnl(sl, ss)
    return float((w.pattern_freq * site).sum()), site


def longdouble_sites(w, P, forced_node=-1, forced_states=None):
    """Per-pattern log-likelihoods of one rate class by tests/resident_reference.py's plain recursion in numpy.longdouble
    without any scaling: its exponent range (x86-64: 80-bit extended, down to 2^-16382) covers every product in this
    suite.  Optionally one node (flat id) pinned to a state per pattern."""
    pin = (forced_node, forced_states) if forced_node >= 0 else None
    return rr.class_sites(w.tree, P, w.leaf_states.T, w.ambig, w.pi, pin).astype(np.float64)


def depth_of(tree):
    L, I = tree.n_leaves, tree.n_internal
    par = np.asarray(tree.flat_parents)
    depth = np.zeros(L + I, dtype=int)
    for n in range(L + I - 2, -1, -1):
        depth[n] = depth[L + par[n]] + 1
    return depth


# ---------------------------------------------------------------------------------------------------------------------
# shared checks
# ---------------------------------------------------------------------------------------------------------------------
def check_lnl(lf, w, mode, P=None):
    """lnL and per-pattern values against the oracle (one rate class: P given; else port.lnl over all classes)."""
    rtol, atol = tol(w, mode)
    lnl, sl, ss = lf.compute(want_sites=True)
    if P is not None:
        ref, site = oracle_sites(w, P)
    else:
        ref, site = port.lnl(w, sparse_storage=sparse(w))
    assert np.isfinite(lnl)
    assert abs(lnl - ref) <= rtol * abs(ref), (lnl, ref)
    assert np.abs(_site_lnl(sl, ss) - site).max() <= atol
    return lnl


def oracle_lnl(w, Qt, P=None, node=None):
    """The oracle's lnL for the rate matrices Qt.  One-class workloads may pass P, the oracle's matrices of w.Qt(): then only
    branch `node`, the one that differs, is exponentiated again."""
    if P is None:
        return port.lnl(w, Qt, sparse_storage=sparse(w))[0]
    P2 = P.copy()
    P2[node] = port.expm(Qt[0, node], sparse(w))
    return oracle_sites(w, P2)[0]


def check_partial(lf, w, mode, node, P=None):
    """Branch `node` changes; only it is passed.  fp64 kernels: bit-identical to a full recomputation; both: the oracle."""
    rtol, _ = tol(w, mode)
    w.tree.t[node] *= 1.6
    Qt = w.Qt()
    for c in range(w.C):
        lf.part.set_matrices(c, [node], Qt[c, node:node + 1])
    part, psl, pss = lf.compute(update_nodes=[node], want_sites=True)
    full, fsl, fss = lf.compute(update_nodes=None, want_sites=True)
    ref = oracle_lnl(w, Qt, P, node)
    w.tree.t[node] /= 1.6
    for c in range(w.C):
        lf.part.set_matrices(c, [node], w.Qt()[c, node:node + 1])
    lf.compute(update_nodes=[node])
    assert abs(part - ref) <= rtol * abs(ref), (node, part, ref)
    if mode == "fp64" or w.D <= 32:
        assert part == full and np.array_equal(psl, fsl) and np.array_equal(pss, fss), node
    else:               # tensor path: a partial plan may fold a node's children in another order (fp32 rounding)
        assert abs(part - full) <= 1e-8 * abs(full)


def check_forced(lf, w, mode, nodes, marginal_node=None, seed=1, P=None):
    """Pinned nodes against port.prune_forced (full and children-only update lists); marginalisation on one node."""
    rtol, atol = tol(w, mode)
    rng = np.random.default_rng(seed)
    L = w.tree.n_leaves
    c = w.C - 1
    if P is None or w.C > 1:
        P = oracle_P(w, c)
    children = w.tree.children()
    base, bl, bs = lf.compute_block(c, want_sites=True)
    for node in nodes:
        fs = rng.integers(0, w.D, size=w.S)
        oL, oS = port.prune_forced(w, P, node, fs)
        ref_site = _site_lnl(np.maximum(oL, 1e-300), oS)
        if w.C == 1 and np.any(oL == 0):
            # The oracle, like the reference, boosts one node by at most ~2^495 (tree.cpp:129,182); an unlikely pinned
            # state at a wide node can fall below that.  There, the long-double recursion is the reference.
            ld = longdouble_sites(w, P, node, fs)
            ref_site = np.where(oL > 0, ref_site, ld)
            oL = np.where(oL > 0, oL, np.isfinite(ld).astype(float))
        ok = oL > 0
        upd = [node] if node < L else children[node - L]
        for u in (None, upd):
            lnl, sl, ss = lf.part.evaluate_forced(c, w.pi, node, fs, update_nodes=u)
            assert np.array_equal(sl > 0, ok), node
            got = _site_lnl(np.maximum(sl, 1e-300), ss)
            assert np.abs(got[ok] - ref_site[ok]).max() <= max(atol, 1e-9), (node, u is None)
            if ok.all():
                ref = (w.pattern_freq * ref_site).sum()
                assert abs(lnl - ref) <= rtol * abs(ref)
            else:
                assert lnl == -np.inf
        again, al, as_ = lf.compute_block(c, update_nodes=upd, want_sites=True)
        if mode == "fp64" or w.D <= 32:
            assert again == base and np.array_equal(al, bl) and np.array_equal(as_, bs)
        else:
            assert abs(again - base) <= 1e-8 * abs(base) and np.array_equal(as_, bs)
    if marginal_node is not None:       # sum over the states of the pinned likelihoods = the likelihood
        tot = np.zeros(w.S)
        for st in range(w.D):
            _, sl, ss = lf.part.evaluate_forced(c, w.pi, marginal_node, np.full(w.S, st),
                                                update_nodes=children[marginal_node - L])
            tot += sl * 2.0 ** (-64.0 * (ss - bs))
        lf.compute_block(c, update_nodes=children[marginal_node - L])
        np.testing.assert_allclose(tot, bl, rtol=max(10 * atol, 1e-9))


def check_branch_cache(lf, w, mode, nodes, P=None):
    """The single-branch shortcut with the branch's matrix changed = a full evaluation with that matrix."""
    rtol, atol = tol(w, mode)
    Qt = w.Qt()
    base = lf.compute()
    for node in nodes:
        lf.part.branch_cache_build(node, w.pi)
        assert abs(lf.part.branch_cache_evaluate(w.class_weights) - base) <= max(rtol, 1e-12) * abs(base)
        for c in range(w.C):
            lf.part.set_matrices(c, [node], (Qt[c, node] * 2.5)[None])
        got, sl, ss = lf.part.branch_cache_evaluate(w.class_weights, want_sites=True)
        full, fl, fs = lf.compute(update_nodes=[node], want_sites=True)
        Q2 = Qt.copy()
        Q2[:, node] *= 2.5
        ref = oracle_lnl(w, Q2, P, node)
        assert abs(got - full) <= max(rtol, 1e-12) * abs(full), (node, got, full)
        assert abs(got - ref) <= rtol * abs(ref)
        assert np.abs(_site_lnl(sl, ss) - _site_lnl(fl, fs)).max() <= max(atol, 1e-9)
        for c in range(w.C):
            lf.part.set_matrices(c, [node], Qt[c, node][None])
        assert lf.compute(update_nodes=[node]) == base or mode == "tc"


def widest_node(tree):
    """The internal node with the most children (flat id), one branch directly under it (an internal child if it has
    one) and all its children."""
    ch = tree.children()
    i = int(np.argmax([len(c) for c in ch]))
    kids = ch[i]
    inner = [c for c in kids if c >= tree.n_leaves]
    return tree.n_leaves + i, (inner[0] if inner else kids[0]), kids


# ---------------------------------------------------------------------------------------------------------------------
# (a) state-count sweep
# ---------------------------------------------------------------------------------------------------------------------
SWEEP = [2, 3, 4, 5, 6, 8, 9, 12, 16, 17, 20, 24, 25, 29, 32, 33, 40, 48, 61, 63, 64]


def sweep_workload(D):
    C = 3 if SWEEP.index(D) % 2 else 1
    w = synth.generic_workload(D, 16, 300, C, seed=41)            # 16 taxa: 29 branches per class (shared powers at Dp 64)
    if w.S % 128 == 0:
        w.leaf_states, w.pattern_freq = w.leaf_states[:, 1:].copy(), w.pattern_freq[1:].copy()
    inject_ambiguity(w, np.random.default_rng(D))
    return w


def expected_kernel(D, mode):
    Dp = pad_states(D)
    if Dp == 64:
        return {"prune64_tc_walk_kernel"} if mode == "tc" else {"prune64_lanes_kernel"}
    if Dp >= 16:
        return {"prune_small_dmma_kernel"}
    return {"prune_small_walk_kernel", "prune_small_walk_ilp_kernel"} if Dp == 4 else {"prune_small_walk_kernel"}


def norm1(A):
    return np.abs(A).sum(axis=0).max()


def edge_matrices(Q):
    """(label, Q*t, atol against the oracle) at the lengths where exp(Qt) is hardest: 0, 1e-8, ||Qt||_1 just below and
    just above 2^0, 2^3 and 2^6, and a saturating length.  Tolerances: 3e-14 without squaring, as for 61 states
    (test_expm_matches_oracle); with squarings those of test_expm_large_rates_and_zero (5e-13, and 1e-10 for the
    saturating length, where 20+ squarings each add rounding of order 1e-16 * 2^k)."""
    n = norm1(Q)
    out = [("zero", Q * 0.0, 0.0), ("1e-8", Q * 1e-8, 3e-14)]
    for p in (0, 3, 6):
        for f, lab in ((1 - 1e-9, "below"), (1 + 1e-9, "above")):
            out.append((f"2^{p} {lab}", Q * (2.0 ** p * f / n), 3e-14 if (p == 0 and f < 1) else 5e-13))
    out.append(("saturating", Q * (4000.0 / n), 1e-10))
    return out


@pytest.mark.parametrize("D,mode", with_modes(SWEEP))
def test_state_count_sweep(D, mode):
    w = sweep_workload(D)
    rtol, atol = tol(w, mode)
    assert w.S % 128 != 0
    lf = LF(w, mode)
    assert lf.part.pruning_kernel in expected_kernel(D, mode)
    lf.set_all_matrices()
    check_lnl(lf, w, mode)
    L, I = w.tree.n_leaves, w.tree.n_internal

    # transition matrices: dense hand-over at the edges (for Dp = 64 after the power table was built: a small batch proportional
    # to the cached direction takes the polynomial, the others the product kernel)
    Q = w.Q_classes[0]
    edges = edge_matrices(Q)
    lf.part.set_matrices(0, np.arange(len(edges)), np.stack([e[1] for e in edges]))
    for b, (label, A, atol_m) in enumerate(edges):
        P = lf.part.read_transition(0, b)
        if label == "zero":
            np.testing.assert_array_equal(P, np.eye(D))
            continue
        np.testing.assert_allclose(P, port.expm(A, False), rtol=0, atol=atol_m, err_msg=label)
        np.testing.assert_allclose(P, scipy.linalg.expm(A), rtol=0, atol=atol_m, err_msg=label)
        assert np.all(P >= 0) and np.abs(P.sum(axis=1) - 1.0).max() <= 1e-14, label
        if label == "saturating":
            np.testing.assert_allclose(P, np.tile(w.pi, (D, 1)), rtol=0, atol=1e-9)
    lf.set_all_matrices()
    dense = {(c, b): lf.part.read_transition(c, b) for c in range(w.C) for b in (0, L, w.tree.n_branches - 1)}
    lnl_dense = lf.compute()

    # partial updates: a leaf branch and an internal branch
    check_partial(lf, w, mode, 1)
    check_partial(lf, w, mode, L + 1)
    # forced states: a leaf, an internal node, the root; marginalisation on an internal node
    check_forced(lf, w, mode, [0, L + I // 2, L + I - 1], marginal_node=L + I // 3)
    # branch cache: a leaf branch, the deepest internal branch, a child of the root
    depth = depth_of(w.tree)
    deepest = max(range(L, L + I - 1), key=lambda n: depth[n])
    root_child = next(n for n in range(L + I - 1) if w.tree.flat_parents[n] == I - 1)
    check_branch_cache(lf, w, mode, sorted({0, deepest, root_child}))

    # conditionals' read-back against the oracle's (which multiplies a row by 2^64 whenever it fell below 2^-64)
    P0 = np.stack([port.expm(q, False) for q in w.Qt()[0]])
    _, _, ocond = port.prune(w, P0, want_cond=True)
    lf.compute(update_nodes=None)
    for inode in range(I):
        cond, e = lf.part.read_conditionals(0, inode)
        rowmax = ocond[inode].max(axis=1, keepdims=True)
        got = cond * np.exp2(e)[:, None]
        k = np.rint(np.log2(rowmax[:, 0] / got.max(axis=1)) / 64.0)
        assert np.all(k >= 0)
        got = got * np.exp2(64.0 * k)[:, None]
        a, r = (1e-12, 1e-9) if (mode == "fp64" or D <= 32) else (3e-6, 3e-5)
        assert np.all(np.abs(got - ocond[inode]) <= a * rowmax + r * ocond[inode]), inode
        assert np.all(cond.max(axis=1) >= 0.5) and np.all(cond.max(axis=1) <= 1.0)
    lf.close()

    # compiled hand-over (generic template: every off-diagonal entry its own formula) = dense hand-over
    lf = LF(w, mode)
    lf.set_template()
    lf.set_all_compiled()
    comp = lf.compute()
    for (c, b), Pd in dense.items():
        np.testing.assert_allclose(lf.part.read_transition(c, b), Pd, rtol=0, atol=1e-14)
    assert abs(comp - lnl_dense) <= 1e-12 * abs(lnl_dense)
    lf.close()

    # impossible patterns (identity matrices, differing leaves) and a NaN in Q
    lf = LF(w, mode)
    for c in range(w.C):
        lf.part.set_matrices(c, lf.all_nodes, np.tile(np.eye(D), (w.tree.n_branches, 1, 1)), engine.MATRIX_TRANS)
    assert lf.compute() == -np.inf
    lf.close()
    lf = LF(w, mode)
    Qt = w.Qt()
    Qt[0, 2, 1, 1] = np.nan
    lf.set_all_matrices(Qt)
    assert np.isnan(lf.compute())
    lf.close()


# ---------------------------------------------------------------------------------------------------------------------
# (b) pattern counts at the edges of a tile: one D per padding bucket
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S", [1, 2, 127, 129, 300])
@pytest.mark.parametrize("D,mode", with_modes([3, 7, 12, 20, 29, 48]))
def test_pattern_count_edges(D, mode, S):
    """S = 300 on 4 states: Sp/128 = 3 is odd, so the two-patterns-per-thread kernel has a dead slot in its last CTA."""
    tree = synth.random_tree(12, 5, mean_t=0.2)
    w = tree_workload(tree, D, 900, seed=5, n_patterns=S)
    lf = LF(w, mode)
    lf.set_all_matrices()
    check_lnl(lf, w, mode, oracle_P(w))
    lf.close()


# ---------------------------------------------------------------------------------------------------------------------
# (c) tree shapes
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D,mode", with_modes([4, 6, 20, 32, 61]))
@pytest.mark.parametrize("shape", list(TREES))
def test_tree_shapes(shape, D, mode):
    tree = flat_tree(TREES[shape], mean_t=0.2, seed=len(shape))
    w = tree_workload(tree, D, 150, seed=9)
    lf = LF(w, mode)
    lf.set_all_matrices()
    P = oracle_P(w)
    check_lnl(lf, w, mode, P)
    node, under, _ = widest_node(tree)
    check_partial(lf, w, mode, under, P)
    check_forced(lf, w, mode, [node], P=P)
    check_branch_cache(lf, w, mode, [under], P)
    lf.close()


# ---------------------------------------------------------------------------------------------------------------------
# (d) kernel variants chosen by the host or by a switch: same results
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [9, 16, 17, 24])
def test_small_dmma_cta_shapes_agree_bitwise(D, monkeypatch):
    """prune_small_dmma_kernel<Dp, 4> and <Dp, 8> do the same arithmetic per pattern (HB2_SMALL_WARPS is read at launch)."""
    w = synth.generic_workload(D, 16, 300, 2, seed=13)
    L, I = w.tree.n_leaves, w.tree.n_internal
    fs = np.random.default_rng(2).integers(0, D, size=w.S)
    out = {}
    for nw in ("4", "8"):
        monkeypatch.setenv("HB2_SMALL_WARPS", nw)
        lf = LF(w, "fp64")
        lf.set_all_matrices()
        out[nw] = (lf.compute(want_sites=True), lf.part.evaluate_forced(1, w.pi, L + I // 2, fs))
        lf.close()
    (a, fa), (b, fb) = out["4"], out["8"]
    assert a[0] == b[0] and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])
    assert fa[0] == fb[0] and np.array_equal(fa[1], fb[1]) and np.array_equal(fa[2], fb[2])
    ref, _ = port.lnl(w, sparse_storage=False)
    assert abs(a[0] - ref) <= 1e-10 * abs(ref)


@pytest.mark.parametrize("D", [2, 3])
def test_small_walk_one_and_two_patterns_per_thread_agree_bitwise(D, monkeypatch):
    """S = 300: Sp/128 = 3 is odd, so the last CTA of the two-patterns-per-thread kernel has a dead slot."""
    w = tree_workload(synth.random_tree(14, 7, mean_t=0.2), D, 2000, seed=7, n_patterns=300)
    kernels = {"1": "prune_small_walk_kernel", "2": "prune_small_walk_ilp_kernel"}
    out = {}
    for ilp in ("1", "2"):
        monkeypatch.setenv("HB2_SMALL_ILP", ilp)
        lf = LF(w, "fp64")
        assert lf.part.pruning_kernel == kernels[ilp]
        lf.set_all_matrices()
        out[ilp] = lf.compute(want_sites=True)
        check_lnl(lf, w, "fp64", oracle_P(w))
        lf.close()
    a, b = out["1"], out["2"]
    assert a[0] == b[0] and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])


WALK_SWITCHES = [{"HB2_WALK_LANES": "1"}, {"HB2_WALK_LANES": "2"}, {"HB2_WALK_LANES": "15"}, {"HB2_WALK_SPLIT_NODES": "0"}]


@pytest.mark.parametrize("mode", ["fp64", "tc"])
@pytest.mark.parametrize("shape", ["poly7", "poly33", "all_internal", "star40"])
def test_walk_plans_do_not_change_results(shape, mode, monkeypatch):
    """fp64 lanes kernel: results do not depend on the plan (lane count, side products), bit for bit.  Tensor walk: within
    1e-8 of its default plan (fp32 rounding of another folding order), and each plan within tolerance of the oracle."""
    w = tree_workload(flat_tree(TREES[shape], mean_t=0.2, seed=3), 61, 300, seed=4)
    P = oracle_P(w)
    lf = LF(w, mode)
    lf.set_all_matrices()
    base = lf.compute(want_sites=True)
    lf.close()
    for sw in WALK_SWITCHES:
        for k, v in sw.items():
            monkeypatch.setenv(k, v)
        lf = LF(w, mode)
        lf.set_all_matrices()
        got = lf.compute(want_sites=True)
        check_lnl(lf, w, mode, P)
        lf.close()
        for k in sw:
            monkeypatch.delenv(k)
        if mode == "fp64":
            assert got[0] == base[0] and np.array_equal(got[1], base[1]) and np.array_equal(got[2], base[2]), sw
        else:
            assert abs(got[0] - base[0]) <= 1e-8 * abs(base[0]), sw


@pytest.mark.parametrize("D", [33, 48, 64])
def test_expm_shared_powers_off_gives_same_matrices(D, monkeypatch):
    """33..64 states other than 61: the shared-powers pipeline (classify, powers, poly) against the product kernel alone."""
    w = synth.generic_workload(D, 16, 100, 3, seed=17)
    Qt = w.Qt()
    mats = {}
    for shared in ("1", "0"):
        monkeypatch.setenv("HB2_EXPM_SHARED", shared)
        lf = LF(w, "fp64")
        lf.set_all_matrices(Qt)
        mats[shared] = np.stack([[lf.part.read_transition(c, b) for b in range(w.tree.n_branches)] for c in range(w.C)])
        lf.close()
    np.testing.assert_allclose(mats["1"], mats["0"], rtol=0, atol=1e-13)


# ---------------------------------------------------------------------------------------------------------------------
# (e) products over the children of a wide node that underflow a double
# ---------------------------------------------------------------------------------------------------------------------
UNDERFLOW = {                         # (leaves, states, mean branch length)
    "codon400": (400, 61, 2.0),
    "nuc1500": (1500, 4, 0.5),
    "rev20_250": (250, 20, 20.0),          # saturated branches: every leaf costs about log2(20) bits
}


def underflow_workload(name):
    L, D, mean_t = UNDERFLOW[name]
    tree = flat_tree(star(L), mean_t=mean_t, seed=11)
    if D != 61:
        if D == 4:
            pi = np.array([0.30, 0.22, 0.24, 0.24])
            Q, meta = synth.hky85_Q(2.0, pi), {"kind": "nuc", "kappa": 2.0}
        else:       # even frequencies: a saturated branch costs log2(D) bits, the most a leaf can cost
            rng = np.random.default_rng(D)
            R = rng.gamma(1.0, 1.0, size=(D, D))
            pi = np.full(D, 1.0 / D)
            Q = (R + R.T) / 2 * pi[None, :]
            Q[np.diag_indices(D)] = 0.0
            Q[np.diag_indices(D)] = -Q.sum(axis=1)
            Q /= -(pi * np.diag(Q)).sum()
            meta = {"kind": "generic"}
        Ps =[[synth._expm_np(Q * t) for t in tree.t[:tree.n_branches]]]
        states = synth._simulate(tree, Ps, pi, np.zeros(200, dtype=np.int64), np.random.default_rng(12))
        ls, freq, s2p = synth.compress(states)
        return synth.Workload(name, tree, D, pi, [Q], np.array([1.0]), ls, np.zeros((0, D)), freq, s2p, None, meta)
    w = tree_workload(tree, D, 200, seed=12)
    w.name = name
    return w


def log2_unscaled_max(w, P):
    """log2 of max over parent states of the product over the root's children, computed in logs (no underflow): what the
    product reaches without any rescaling inside the node."""
    logv = np.zeros((w.S, w.D))
    for leaf in range(w.tree.n_leaves):
        logv += np.log(np.maximum(P[leaf][:, w.leaf_states[leaf]].T, 1e-300))
    return logv.max(axis=1) / np.log(2.0)


@pytest.mark.parametrize("name,mode", [(n, m) for n in UNDERFLOW for m in (["fp64", "tc"] if UNDERFLOW[n][1] > 32 else ["fp64"])])
def test_wide_node_underflow(name, mode):
    w = underflow_workload(name)
    P = oracle_P(w)
    m = log2_unscaled_max(w, P)
    assert np.mean(m < -1022) > 0.5, np.median(m)      # the unscaled product really leaves the double range
    lf = LF(w, mode)
    lf.set_all_matrices()
    if name != "nuc1500":
        check_lnl(lf, w, mode, P)
    else:
        # The oracle, like the reference, boosts one node by at most sqrt(DBL_MAX * 1e-10) ~ 2^495 (tree.cpp:129,182): a
        # product of 2^-1750 leaves it at 0 and lnL = -inf.  The engine's exponent has no such cap, so it is held to the
        # plain long-double recursion on the same matrices instead.
        assert port.prune(w, P)[0].min() == 0.0
        site = longdouble_sites(w, P)
        ref = float((w.pattern_freq * site).sum())
        rtol, atol = tol(w, mode)
        lnl, sl, ss = lf.compute(want_sites=True)
        assert np.isfinite(lnl) and abs(lnl - ref) <= rtol * abs(ref), (lnl, ref)
        assert np.abs(_site_lnl(sl, ss) - site).max() <= atol
    lf.close()


def test_wide_node_underflow_batched_site_likelihoods():
    """hb2_batch_site_likelihoods (prune_batch_kernel) on the 400-leaf codon star: one-pattern likelihoods = the oracle's."""
    w = underflow_workload("codon400")
    P = oracle_P(w)
    assert np.mean(log2_unscaled_max(w, P) < -1022) > 0.5
    lf = LF(w, "fp64")
    lf.set_template()
    vals = w.compiled_values()[0]
    pats = np.arange(min(w.S, 24))
    got = lf.part.batch_site_likelihoods(pats, np.broadcast_to(vals, (len(pats),) + vals.shape), w.pi)
    lf.close()
    for i, p in enumerate(pats):
        w1 = synth.Workload("one", w.tree, w.D, w.pi, w.Q_classes, w.class_weights, w.leaf_states[:, p:p + 1], w.ambig,
                            np.array([1]), np.array([0]))
        sl, ss = port.prune(w1, P)
        ref = float(_site_lnl(sl, ss)[0])
        assert np.isfinite(got[i]) and abs(got[i] - ref) <= 1e-10 * abs(ref) + 1e-12, (i, got[i], ref)
