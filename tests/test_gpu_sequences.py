"""GPU suite (pytest -m gpu): non-reversible models, root vectors other than the model's frequencies, and long seeded
optimiser-shaped call sequences, against the oracle.

For a reversible model with its stationary vector at the root, lnL does not depend on where the root is or which way a
branch is read, so an error that amounts to re-rooting the tree or reading a branch upside down passes every test built on
such models.  Here every generator is non-reversible and every root vector differs from the model's frequencies;
tests/test_sequence_reference.py shows that both errors then move lnL by at least 1e-3 relative.  The engine claims not
to need reversibility (the branch cache propagates outside vectors with the transposed matrices) and takes the root
vector as an independent input of every entry point; these tests check both claims on every kernel family.

The sequences interleave what an optimiser driving the engine does -- per-class evaluations with their dirty lists,
root-vector and weight changes with empty lists, pinned nodes with their recompute lists, branch caches, batched site
likelihoods, conditionals' read-back, a partition re-created from recycled blocks -- and check every step against
tests/sequence_cases.SequenceModel (the oracle from scratch) and against a twin partition that always prunes the whole
tree.  Tolerances are those of test_gpu_parity.py."""
import collections

import numpy as np
import pytest
import scipy.linalg

from hyphy_b200 import LikelihoodFunction, engine
from oracle import port
from tests import handover_cases as hc
from tests import sequence_cases as sc
from tests.test_gpu_shapes import expected_kernel

pytestmark = pytest.mark.gpu

MODES = {"fp64": (engine.FLAG_FORCE_FP64, 1e-10, 1e-8),     # flags, lnL rtol, per-pattern atol
         "tc": (engine.FLAG_DEFAULT, 1e-7, 1e-5)}
RESIDENT_RTOL = {"fp64": 1e-12, "tc": 1e-9}


@pytest.fixture(scope="module", autouse=True)
def _need_gpu(engine_lib):
    assert engine.device_count() > 0, "GPU tests need a CUDA device (no fallback exists)"


def LF(w, mode):
    return LikelihoodFunction(w, flags=MODES[mode][0])


def tol(D, mode):
    return MODES["tc"][1:] if (mode == "tc" and D > 32) else MODES["fp64"][1:]


def bitwise(D, mode):
    """fp64 kernels: a partial evaluation equals a full one bit for bit; the tensor walk may fold in another order."""
    return mode == "fp64" or D <= 32


def with_modes(names):
    return [(n, "fp64") for n in names] + [(n, "tc") for n in names if sc.model(n).D > 32]


def check_P(part, sm, c, b, label):
    P = part.read_transition(c, b)
    err = float(np.abs(P - sm.P[c, b]).max())
    assert err <= sm.atol[c, b], f"{label}: class {c} branch {b}: |P - oracle| = {err:.3e} > {sm.atol[c, b]:.0e}"
    rs = float(np.abs(P.sum(axis=1) - 1.0).max())
    assert rs <= 1e-14, f"{label}: class {c} branch {b}: row sums off by {rs:.3e}"
    return P


def check_value(label, got, ref, D, mode, sites=None, ref_sites=None):
    rtol, atol = tol(D, mode)
    assert np.isfinite(got) and abs(got - ref) <= rtol * abs(ref), f"{label}: lnL {got!r}, oracle {ref!r}, rel {abs(got - ref) / abs(ref):.2e}"
    if sites is not None:
        err = float(np.abs(sites - ref_sites).max())
        assert err <= atol, f"{label}: per-pattern error {err:.2e}"


def check_conditionals(part, sm, c, inode, mode, label):
    """Read-back against the oracle's conditionals, which multiply a row by 2^64 whenever it fell below 2^-64."""
    ocond = sm.conditionals(c)[inode]
    cond, e = part.read_conditionals(c, inode)
    rowmax = ocond.max(axis=1, keepdims=True)
    got = cond * np.exp2(e)[:, None]
    k = np.rint(np.log2(rowmax[:, 0] / got.max(axis=1)) / 64.0)
    assert np.all(k >= 0), label
    got = got * np.exp2(64.0 * k)[:, None]
    a, r = (1e-12, 1e-9) if bitwise(sm.w.D, mode) else (3e-6, 3e-5)
    bad = np.abs(got - ocond) > a * rowmax + r * ocond
    assert not bad.any(), f"{label}: class {c} node {inode}: {int(bad.sum())} conditionals off"


def sites_of(sl, ss):
    return hc.site_lnl(sl, ss)


# ---------------------------------------------------------------------------------------------------------------------
# 1. non-reversible models on every kernel family
# ---------------------------------------------------------------------------------------------------------------------
NONREV = ["nrm4", "rand8", "rand20", "rand24", "codon61", "drift64"]


@pytest.mark.parametrize("name,mode", with_modes(NONREV))
def test_nonreversible_model(name, mode):
    """Transition matrices (shared-powers and general path, 0 to lengths that need squarings), lnL and per-pattern values,
    partial = full, pinned nodes and conditionals, at a non-equilibrium root.  Class 0 is handed over compiled, class 1
    dense: both are proportional over all 29 branches, so at 33..64 states each builds a shared-powers table."""
    m = sc.model(name, 2, seed=1)
    w = sc.workload(m, 16, 200, seed=3)
    D, L, I = w.D, w.tree.n_leaves, w.tree.n_internal
    root = sc.root_vectors(w, 3)["dirichlet"]
    sm = sc.SequenceModel(w, root, w.class_weights)
    lf = LF(w, mode)
    p = lf.part
    assert p.pruning_kernel in expected_kernel(D, mode)
    m.tmpl.define(p, 0)
    t = w.tree.t[:sm.B]
    nodes = np.arange(sm.B)
    p.set_matrices_compiled(0, nodes, m.x[0][None, :] * t[:, None])
    p.set_matrices(1, nodes, m.Q[1][None] * t[:, None, None])
    for c in range(2):
        for b in nodes:
            sm.set_Q(c, b, m.Q[c] * t[b])
    for c in range(2):
        for b in nodes:
            check_P(p, sm, c, b, f"{name} start")
    lnl, sl, ss = p.evaluate_classes(w.class_weights, root, want_sites=True)
    ref, ref_sites = sm.lnl()
    check_value(f"{name} start", lnl, ref, D, mode, sites_of(sl, ss), ref_sites)

    # transition matrices at the edges.  Class 0: compiled values proportional to the direction its table was built from,
    # six entries (fewer than a group needs for a table of its own): at 33..64 states each is compared with the cached
    # direction of the same kind and takes the shared-powers polynomial.  Class 1: a different generator per branch, which
    # is proportional to nothing (the general path).
    n = hc.inf_norm(m.Q[0])
    lengths = [0.0, 1e-8, 0.3 / n, 2.0 / n, 30.0 / n, 600.0 / n]
    G = sc.random_Q(D, 99)[0]
    edge = np.arange(len(lengths))
    p.set_matrices_compiled(0, edge, np.stack([m.x[0] * s for s in lengths]))
    gen = np.stack([(m.Q[1] + 0.2 * (k + 1) * G) * s for k, s in enumerate(lengths)])
    p.set_matrices(1, edge, gen)
    for k, s in enumerate(lengths):
        A0 = m.tmpl.Q(m.x[0] * s)
        sm.set_Q(0, k, A0, shared_powers=D > 32)
        sm.set_Q(1, k, gen[k])
        for c, A in ((0, A0), (1, gen[k])):
            P = check_P(p, sm, c, k, f"{name} length {s:.3g}")
            if s == 0.0:
                np.testing.assert_array_equal(P, np.eye(D))
            else:
                np.testing.assert_allclose(P, scipy.linalg.expm(A), rtol=0, atol=hc.p_atol(A), err_msg=f"{name} scipy {s:.3g}")
    lnl, sl, ss = p.evaluate_classes(w.class_weights, root, update_nodes=edge, want_sites=True)
    ref, ref_sites = sm.lnl()
    check_value(f"{name} after the edge lengths", lnl, ref, D, mode, sites_of(sl, ss), ref_sites)

    # partial = full: a leaf branch and an internal branch
    for node in (len(lengths) + 1, L + 1):
        for c in range(2):
            A = m.Q[c] * (t[node] * 1.7)
            p.set_matrices(c, [node], A[None])
            sm.set_Q(c, node, A)
        part, psl, pss = p.evaluate_classes(w.class_weights, root, update_nodes=[node], want_sites=True)
        full, fsl, fss = p.evaluate_classes(w.class_weights, root, want_sites=True)
        check_value(f"{name} partial, node {node}", part, sm.lnl()[0], D, mode)
        if bitwise(D, mode):
            assert part == full and np.array_equal(psl, fsl) and np.array_equal(pss, fss), f"{name} node {node}: {part!r} != {full!r}"
        else:
            assert abs(part - full) <= 1e-8 * abs(full), f"{name} node {node}: {part!r}, {full!r}"

    # pinned nodes: a leaf, an internal node, the root; then every node's conditionals
    rng = np.random.default_rng(4)
    children = w.tree.children()
    for node in (0, L + I // 2, L + I - 1):
        fs = rng.integers(0, D, size=w.S)
        ref_site, ok = sm.forced_sites(1, node, fs)
        for u in (None, [node] if node < L else children[node - L]):
            lnl, sl, ss = p.evaluate_forced(1, root, node, fs, update_nodes=u)
            assert np.array_equal(sl > 0, ok), f"{name} pinned {node}"
            got = sites_of(np.maximum(sl, 1e-300), ss)
            assert np.abs(got[ok] - ref_site[ok]).max() <= max(tol(D, mode)[1], 1e-9), f"{name} pinned {node}"
            if ok.all():
                check_value(f"{name} pinned {node}", lnl, float((w.pattern_freq * ref_site).sum()), D, mode)
        p.evaluate(1, root, update_nodes=[node] if node < L else children[node - L])
    p.evaluate_classes(w.class_weights, root)
    for c in range(2):
        for inode in range(I):
            check_conditionals(p, sm, c, inode, mode, name)
    lf.close()


# ---------------------------------------------------------------------------------------------------------------------
# 2. the root vector is an input of its own on every entry point
# ---------------------------------------------------------------------------------------------------------------------
ROOTS = ["nrm4", "rand20", "codon61", "drift64"]


@pytest.mark.parametrize("name,mode", with_modes(ROOTS))
def test_root_vector_on_every_entry_point(name, mode, request):
    """A Dirichlet root vector, one with zeros and a point mass, each different from the model's stationary vector, on
    evaluate, evaluate_classes, evaluate_forced, the branch cache (leaf, internal and root-child branch), batched site
    likelihoods and hb2_time_resident; a root-vector change with an empty update list equals a full recomputation."""
    m = sc.model(name, 3, seed=2)
    w = sc.workload(m, 16, 150, seed=6)
    D, L, I = w.D, w.tree.n_leaves, w.tree.n_internal
    roots = sc.root_vectors(w, 8)
    sm = sc.SequenceModel(w, roots["dirichlet"], w.class_weights)
    lf = LF(w, mode)
    p = lf.part
    m.tmpl.define(p, 0)
    t = w.tree.t[:sm.B]
    nodes = np.arange(sm.B)
    for c in range(w.C):
        p.set_matrices_compiled(c, nodes, m.x[c][None, :] * t[:, None])
        for b in nodes:
            sm.set_Q(c, b, m.Q[c] * t[b])
    wts = w.class_weights
    p.evaluate_classes(wts, sm.root)
    rng = np.random.default_rng(9)
    root_child = next(n for n in range(L + I - 1) if w.tree.flat_parents[n] == I - 1 and n >= L)
    deep = next(n for n in range(L, L + I - 1) if n != root_child and w.tree.flat_parents[n] != I - 1)
    for label, r in roots.items():
        sm.set_root(r)
        # an empty list after another root vector: only the root vector changed
        lnl, sl, ss = p.evaluate_classes(wts, r, update_nodes=[], want_sites=True)
        full, fsl, fss = p.evaluate_classes(wts, r, want_sites=True)
        ref, ref_sites = sm.lnl()
        check_value(f"{label}: evaluate_classes, empty list", lnl, ref, D, mode, sites_of(sl, ss), ref_sites)
        if bitwise(D, mode):
            assert lnl == full and np.array_equal(sl, fsl), f"{label}: empty list {lnl!r} != full {full!r}"
        for c in range(w.C):
            got, sl, ss = p.evaluate(c, r, update_nodes=[], want_sites=True)
            ref, ref_sites = sm.class_lnl(c)
            check_value(f"{label}: evaluate class {c}", got, ref, D, mode, sites_of(sl, ss), ref_sites)
        fs = rng.integers(0, D, size=w.S)
        for node in (1, L + 2):
            ref_site, ok = sm.forced_sites(2, node, fs)
            got, sl, ss = p.evaluate_forced(2, r, node, fs)
            assert np.array_equal(sl > 0, ok), f"{label}: pinned {node}"
            assert np.abs(sites_of(np.maximum(sl, 1e-300), ss)[ok] - ref_site[ok]).max() <= max(tol(D, mode)[1], 1e-9), f"{label}: pinned {node}"
        p.evaluate_classes(wts, roots["dirichlet"])        # d_pi now holds another vector than the cache's
        # branch cache built under root vector r, on a leaf branch, an internal branch and a child of the root
        for node in (0, deep, root_child):
            p.branch_cache_build(node, r)
            got = p.branch_cache_evaluate(wts)
            check_value(f"{label}: branch cache {node}, unchanged", got, sm.lnl()[0], D, mode)
            old = sm.P[:, node].copy(), sm.atol[:, node].copy()
            for c in range(w.C):
                A = m.Q[c] * (t[node] * 2.5)
                p.set_matrices(c, [node], A[None])
                sm.set_Q(c, node, A)
            got, sl, ss = p.branch_cache_evaluate(wts, want_sites=True)
            ref, ref_sites = sm.lnl()
            check_value(f"{label}: branch cache {node}", got, ref, D, mode, sites_of(sl, ss), ref_sites)
            for c in range(w.C):
                p.set_matrices_compiled(c, [node], (m.x[c] * t[node])[None])
                sm.set_P(c, node, old[0][c], old[1][c])
            p.evaluate_classes(wts, roots["dirichlet"], update_nodes=[node])
        if D > 32:
            sets = 6
            V = np.stack([m.x[0][None, :] * (t * (0.6 + 0.2 * s))[:, None] for s in range(sets)])
            pattern_of = np.arange(sets) * 7 % w.S
            out = p.batch_site_likelihoods(pattern_of, V, r)
            for s in range(sets):
                P = np.stack([hc.oracle_P(m.tmpl.Q(V[s, b])) for b in nodes])
                refs = hc.site_lnl(*port.prune(sm.rooted(), P))[pattern_of[s]]
                assert abs(out[s] - refs) <= 1e-10 * abs(refs), f"{label}: batched set {s}: {out[s]!r}, oracle {refs!r}"
        _, _, res = p.time_resident(wts, r, iters=1)
        lnl = p.evaluate_classes(wts, r)
        request.node.user_properties.append((f"{label}: resident bit-identical", repr(res == lnl)))
        assert abs(res - lnl) <= RESIDENT_RTOL[mode] * abs(lnl), f"{label}: resident {res!r}, compute {lnl!r}"
        check_value(f"{label}: after hb2_time_resident", lnl, sm.lnl()[0], D, mode)
    lf.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3. optimiser-shaped sequences
# ---------------------------------------------------------------------------------------------------------------------
class Sequence:
    """One partition driven like an optimiser drives it, a twin that always prunes the whole tree, and the SequenceModel
    both must agree with.  The twin holds the main partition's transition matrices, read back after the main partition
    has used them: two partitions may exponentiate the same input by different paths (a shared-powers table cached in one
    and not in the other) and differ in the last bit.  Every read-back is held to the oracle."""

    KINDS = ("dense", "compiled", "trans", "mixture")

    def __init__(self, name, mode, seed, n_taxa=40, n_sites=100, C=3):
        self.name, self.mode, self.seed = name, mode, seed
        self.rng = np.random.default_rng(seed)
        self.m = sc.model(name, C, seed=seed)
        self.w = w = sc.workload(self.m, n_taxa, n_sites, seed=seed + 1)
        self.D, self.C, self.L, self.I = w.D, C, w.tree.n_leaves, w.tree.n_internal
        self.B = w.tree.n_branches
        self.roots = list(sc.root_vectors(w, seed).values())
        self.sm = sc.SequenceModel(w, self.roots[0], w.class_weights)
        self.main, self.twin = self._part(), LF(w, mode)
        self.t = np.tile(w.tree.t[:self.B], (C, 1))
        self.dirty = [set() for _ in range(C)]
        self.unsynced = set()                  # (class, branch) slots whose matrix the twin does not hold yet
        self.ops = collections.deque(maxlen=10)
        self.step = 0
        for c in range(C):
            self.hand(c, np.arange(self.B), "compiled")

    def _part(self):
        lf = LF(self.w, self.mode)
        self.m.tmpl.define(lf.part, 0)
        return lf

    def fail(self, msg):
        return f"seed {self.seed} step {self.step}: {msg}; last operations: {list(self.ops)}"

    # -- hand-overs ------------------------------------------------------------------------------------------------------
    def hand(self, c, nodes, kind):
        nodes = np.asarray(nodes, dtype=np.int64)
        m, t = self.m, self.t[c, nodes]
        if kind == "compiled":
            V = m.x[c][None, :] * t[:, None]
            self.main.part.set_matrices_compiled(c, nodes, V)
            for b, v in zip(nodes, V):
                self.sm.set_Q(c, b, m.tmpl.Q(v))
        elif kind == "dense":
            A = m.Q[c][None] * t[:, None, None]
            self.main.part.set_matrices(c, nodes, A)
            for b, a in zip(nodes, A):
                self.sm.set_Q(c, b, a)
        elif kind == "trans":
            P = np.stack([hc.oracle_P(m.Q[c] * tb) for tb in t])
            self.main.part.set_matrices(c, nodes, P, engine.MATRIX_TRANS)
            for b, pb in zip(nodes, P):
                self.sm.set_P(c, b, pb)
        else:                                  # two components: this class's generator and the next class's
            M = np.stack([np.stack([m.Q[c] * tb, m.Q[(c + 1) % self.C] * (0.5 * tb)]) for tb in t])
            wts = np.tile([0.7, 0.3], (len(nodes), 1))
            self.main.part.set_mixture_matrices(c, nodes, M, wts)
            for b, mb in zip(nodes, M):
                self.sm.set_mixture(c, b, mb, [0.7, 0.3])
        self.dirty[c] |= set(int(b) for b in nodes)
        self.unsynced |= {(c, int(b)) for b in nodes}

    def sync_twin(self):
        """Called after the main partition has evaluated (its staged matrices are flushed)."""
        for c in range(self.C):
            nodes = sorted(b for cc, b in self.unsynced if cc == c)
            if nodes:
                P = np.stack([check_P(self.main.part, self.sm, c, b, self.fail("read-back")) for b in nodes])
                self.twin.part.set_matrices(c, nodes, P, engine.MATRIX_TRANS)
        self.unsynced = set()

    def new_matrices(self, nodes=None, classes=None):
        classes = classes if classes is not None else sorted(self.rng.choice(self.C, size=self.rng.integers(1, self.C + 1), replace=False))
        kind = self.KINDS[self.rng.integers(len(self.KINDS))]
        if nodes is None:
            nodes = self.rng.choice(self.B, size=self.rng.integers(1, 7), replace=False)
        for c in classes:
            self.t[c, nodes] *= self.rng.uniform(0.6, 1.6, size=len(nodes))
            self.hand(int(c), nodes, kind)
        return kind, list(map(int, classes)), sorted(map(int, nodes))

    # -- evaluations ----------------------------------------------------------------------------------------------------
    def compare(self, label, got, twin, ref):
        lnl, sl, ss = got
        check_value(self.fail(label), lnl, ref[0], self.D, self.mode, sites_of(sl, ss), ref[1])
        if bitwise(self.D, self.mode):
            dl, ds = np.flatnonzero(sl != twin[1]), np.flatnonzero(ss != twin[2])
            if lnl != twin[0] or len(dl) or len(ds):
                raise AssertionError(self.fail(
                    f"{label}: {lnl!r}, twin (whole tree) {twin[0]!r}; siteL differs at {dl[:5].tolist()} "
                    f"({sl[dl[:3]].tolist()} vs {twin[1][dl[:3]].tolist()}), siteScale at {ds[:5].tolist()}"))
        else:
            assert abs(lnl - twin[0]) <= 1e-8 * abs(twin[0]), self.fail(f"{label}: {lnl!r}, twin (whole tree) {twin[0]!r}")
        return lnl

    def eval_class(self, c):
        upd = sorted(self.dirty[c])
        got = self.main.part.evaluate(c, self.sm.root, update_nodes=upd, want_sites=True)
        self.sync_twin()
        twin = self.twin.part.evaluate(c, self.sm.root, want_sites=True)
        self.dirty[c] = set()
        return self.compare(f"class {c}, {len(upd)} dirty", got, twin, self.sm.class_lnl(c))

    def eval_all(self, upd=None):
        upd = sorted(set().union(*self.dirty)) if upd is None else upd
        got = self.main.part.evaluate_classes(self.sm.weights, self.sm.root, update_nodes=upd, want_sites=True)
        self.sync_twin()
        twin = self.twin.part.evaluate_classes(self.sm.weights, self.sm.root, want_sites=True)
        self.dirty = [set() for _ in range(self.C)]
        return self.compare(f"all classes, {len(upd)} dirty", got, twin, self.sm.lnl())

    # -- operations -----------------------------------------------------------------------------------------------------
    def op_matrices(self):
        what = self.new_matrices()
        if self.rng.random() < 0.5:
            for c in sorted(set(what[1])):
                self.eval_class(c)
        else:
            self.eval_all()
        return f"matrices {what}"

    def op_root(self):
        if self.rng.random() < 0.5:
            self.sm.set_root(self.roots[self.rng.integers(len(self.roots))] if self.rng.random() < 0.3
                             else self.rng.dirichlet(np.full(self.D, 1.0)))
            what = "root vector"
        else:
            self.sm.weights = self.rng.dirichlet(np.full(self.C, 2.0))
            what = "weights"
        self.eval_all(upd=[] if not any(self.dirty) else None)
        return f"{what}, empty list"

    def op_forced(self):
        c = int(self.rng.integers(self.C))
        node = int(self.rng.integers(self.L + self.I))
        fs = self.rng.integers(0, self.D, size=self.w.S)
        rec = [node] if node < self.L else self.w.tree.children()[node - self.L]
        upd = sorted(self.dirty[c] | set(rec))
        lnl, sl, ss = self.main.part.evaluate_forced(c, self.sm.root, node, fs, update_nodes=upd)
        self.sync_twin()
        tl, tsl, tss = self.twin.part.evaluate_forced(c, self.sm.root, node, fs)
        # An unlikely pinned state makes a pattern's likelihood hang on the smallest entries of P, whose relative error
        # (an absolute 3e-14 on entries near 1e-11) the oracle's matrices do not share: the pinned values are held to the
        # oracle's pruning of the engine's own matrices, which sync_twin held to the oracle's.
        P = np.stack([self.main.part.read_transition(c, b) for b in range(self.B)])
        sl0, ss0 = port.prune_forced(self.sm.rooted(), P, node, fs)
        ref, ok = sites_of(np.maximum(sl0, 1e-300), ss0), sl0 > 0
        assert np.array_equal(sl > 0, ok), self.fail(f"pinned node {node} class {c}: impossible patterns differ")
        err = float(np.abs(sites_of(np.maximum(sl, 1e-300), ss)[ok] - ref[ok]).max()) if ok.any() else 0.0
        assert err <= max(tol(self.D, self.mode)[1], 1e-9), self.fail(f"pinned node {node} class {c}: per-pattern error {err:.2e}")
        if bitwise(self.D, self.mode):
            assert np.array_equal(sl, tsl) and np.array_equal(ss, tss), self.fail(f"pinned node {node} class {c}: twin differs")
        self.dirty[c] = set(rec)
        self.eval_class(c)                  # the host's recompute list
        return f"pinned node {node} class {c}"

    def op_branch_cache(self):
        self.eval_all()
        node = int(self.rng.integers(self.B))
        if self.rng.random() < 0.5:
            self.sm.set_root(self.rng.dirichlet(np.full(self.D, 1.0)))
        self.main.part.branch_cache_build(node, self.sm.root)
        wts = self.sm.weights
        for k in range(int(self.rng.integers(1, 4))):
            self.new_matrices(nodes=[node], classes=range(self.C))
            got, sl, ss = self.main.part.branch_cache_evaluate(wts, want_sites=True)
            self.sync_twin()
            twin = self.twin.part.evaluate_classes(wts, self.sm.root, want_sites=True)
            rtol, atol = tol(self.D, self.mode)
            ref, ref_sites = self.sm.lnl()
            check_value(self.fail(f"branch cache {node}, matrix {k}"), got, ref, self.D, self.mode, sites_of(sl, ss), ref_sites)
            assert abs(got - twin[0]) <= max(rtol, 1e-12) * abs(twin[0]), self.fail(f"branch cache {node}: {got!r}, twin {twin[0]!r}")
        if self.rng.random() < 0.3:         # another branch's matrix arrives: the cache must refuse
            other = (node + 1 + int(self.rng.integers(self.B - 1))) % self.B
            self.new_matrices(nodes=[other], classes=[0])
            with pytest.raises(engine.EngineError, match="branch cache holds node"):
                self.main.part.branch_cache_evaluate(wts)
        self.eval_all()
        return f"branch cache {node}"

    def op_batch(self):
        before = self.eval_all()
        r = self.rng.dirichlet(np.full(self.D, 1.0))
        t = self.t[0]
        V = np.stack([self.m.x[0][None, :] * (t * f)[:, None] for f in (0.7, 1.3)])
        pattern_of = self.rng.integers(0, self.w.S, size=2)
        out = self.main.part.batch_site_likelihoods(pattern_of, V, r)
        for s in range(2):
            P = np.stack([hc.oracle_P(self.m.tmpl.Q(V[s, b])) for b in range(self.B)])
            ref = hc.site_lnl(*port.prune(sc.with_root(self.w, r), P))[pattern_of[s]]
            assert abs(out[s] - ref) <= 1e-10 * abs(ref), self.fail(f"batched set {s}: {out[s]!r}, oracle {ref!r}")
        after = self.main.part.evaluate_classes(self.sm.weights, self.sm.root, update_nodes=[])
        same = after == before if bitwise(self.D, self.mode) else abs(after - before) <= 1e-8 * abs(before)
        assert same, self.fail(f"evaluation after batched site likelihoods {after!r}, before {before!r}")
        return "batched site likelihoods"

    def op_conditionals(self):
        c = int(self.rng.integers(self.C))
        if self.dirty[c]:
            self.eval_class(c)
        inode = int(self.rng.integers(self.I))
        check_conditionals(self.main.part, self.sm, c, inode, self.mode, self.fail("conditionals"))
        return f"conditionals class {c} node {inode}"

    def op_recreate(self):
        """The main partition is destroyed and re-created from recycled blocks and carries on: partial evaluations, branch
        caches and read-backs then rest on that memory.  Before, the twin's blocks are filled with the conditionals of
        other matrices and freed too, so what the new partition may receive holds wrong values, not stale right ones.  It
        gets the old main partition's transition matrices, read back."""
        nodes = np.arange(self.B)
        P = [np.stack([self.main.part.read_transition(c, b) for b in nodes]) for c in range(self.C)]
        flat = np.full((self.B, self.D, self.D), 1.0 / self.D)
        for c in range(self.C):
            self.twin.part.set_matrices(c, nodes, flat, engine.MATRIX_TRANS)
        self.twin.part.evaluate_classes(self.sm.weights, self.sm.root)
        self.twin.close()
        self.main.close()
        self.main = self._part()
        self.twin = LF(self.w, self.mode)
        for c in range(self.C):
            self.main.part.set_matrices(c, nodes, P[c], engine.MATRIX_TRANS)
            self.dirty[c] = set(range(self.B))
        self.unsynced = {(c, b) for c in range(self.C) for b in range(self.B)}
        self.eval_all()
        return "main partition re-created"

    def run(self, steps):
        ops = [(self.op_matrices, 0.40), (self.op_root, 0.14), (self.op_forced, 0.12), (self.op_branch_cache, 0.10),
               (self.op_conditionals, 0.10), (self.op_recreate, 0.05)]
        if self.D > 32:
            ops.append((self.op_batch, 0.10))
        fns, pr = zip(*ops)
        pr = np.asarray(pr) / sum(pr)
        self.ops.append("start")
        self.eval_all(upd=None)
        for self.step in range(1, steps + 1):
            fn = fns[self.rng.choice(len(fns), p=pr)]
            self.ops.append(fn.__name__[3:])
            self.ops[-1] = fn()

    def close(self):
        self.main.close()
        self.twin.close()


SEQUENCES = [("nrm4", "fp64", 11), ("rand20", "fp64", 12), ("codon61", "fp64", 13), ("codon61", "tc", 14)]


@pytest.mark.parametrize("name,mode,seed", SEQUENCES)
def test_optimiser_sequence(name, mode, seed):
    """160 seeded random steps on a 40-leaf tree with 3 rate classes, one sequence per kernel family (small walk, small
    DMMA, fp64 lanes, tensor walk)."""
    s = Sequence(name, mode, seed)
    assert s.main.part.pruning_kernel in expected_kernel(s.D, mode)
    try:
        s.run(160)
    finally:
        s.close()


PLAN_CASE = ("codon61", 3, 21, 16, 1600, 22)      # model, classes, model seed, taxa, sites, workload seed


@pytest.mark.parametrize("mode", ["fp64", "tc"])
def test_walk_plan_across_class_counts(mode):
    """One class and all three classes pruned in turn over the same dirty set.  At 1400+ patterns the lane count of the
    fp64 lanes and tensor walk kernels (co-resident CTAs over classes x pattern tiles, at most 8) differs between the two,
    so a walk plan cached for one class count must not be replayed for the other.  Each evaluation against the oracle and
    a twin partition that prunes the whole tree from the main partition's matrices, read back (as in Sequence)."""
    name, C, mseed, taxa, sites, wseed = PLAN_CASE
    m = sc.model(name, C, seed=mseed)
    w = sc.workload(m, taxa, sites, seed=wseed)
    assert w.S > 1408                                       # 12 tiles of 128 patterns, 48 of 32
    root = sc.root_vectors(w, 5)["dirichlet"]
    sm = sc.SequenceModel(w, root, w.class_weights)
    main, twin = LF(w, mode), LF(w, mode)
    rng = np.random.default_rng(23)
    t = np.tile(w.tree.t[:sm.B], (C, 1))
    nodes = np.arange(sm.B)
    dirty = list(range(0, w.tree.n_leaves, 2))               # eight leaves: their parents and the paths to the root

    def hand(ids):
        for c in range(C):
            A = m.Q[c][None] * t[c, ids][:, None, None]
            main.part.set_matrices(c, ids, A)
            for b, a in zip(ids, A):
                sm.set_Q(c, b, a)

    def sync(ids, label):
        for c in range(C):
            twin.part.set_matrices(c, ids, np.stack([check_P(main.part, sm, c, b, label) for b in ids]), engine.MATRIX_TRANS)

    def same(label, got, tw, ref):
        check_value(label, got[0], ref[0], w.D, mode, sites_of(got[1], got[2]), ref[1])
        if mode == "fp64":
            assert got[0] == tw[0] and np.array_equal(got[1], tw[1]), f"{label}: {got[0]!r}, twin {tw[0]!r}"
        else:
            assert abs(got[0] - tw[0]) <= 1e-8 * abs(tw[0]), f"{label}: {got[0]!r}, twin {tw[0]!r}"

    try:
        hand(nodes)
        main.part.evaluate_classes(w.class_weights, root)
        sync(nodes, "start")
        for r in range(6):
            t[:, dirty] *= rng.uniform(0.7, 1.4, size=(C, len(dirty)))
            hand(dirty)
            if r % 2:
                got = main.part.evaluate_classes(w.class_weights, root, dirty, want_sites=True)
                sync(dirty, f"round {r}")
                same(f"round {r}: all classes", got, twin.part.evaluate_classes(w.class_weights, root, want_sites=True), sm.lnl())
            else:
                for c in range(C):
                    got = main.part.evaluate(c, root, dirty, want_sites=True)
                    sync(dirty, f"round {r}")
                    same(f"round {r}: class {c}", got, twin.part.evaluate(c, root, want_sites=True), sm.class_lnl(c))
    finally:
        main.close()
        twin.close()
