"""CPU suite: the references of tests/test_gpu_sequences.py (built by tests/sequence_cases.py).

The generators there are not reversible, the oracle's exponential and pruning hold on them against scipy and a
long-double recursion, the algebra behind the branch cache holds without reversibility, and -- what makes the GPU tests
able to see re-rooting and orientation errors at all -- moving the root, or putting the stationary vector where the root
vector belongs, moves lnL by far more than the tensor path's tolerance."""
import numpy as np
import pytest
import scipy.linalg

from oracle import port
from tests import handover_cases as hc
from tests import sequence_cases as sc
from tests import test_gpu_sequences as T
from tests.test_gpu_shapes import depth_of, longdouble_sites

MODELS = ["nrm4", "rand8", "rand20", "rand24", "codon61", "drift64"]
TC_RTOL = 1e-7


def _workload(name, C=2):
    m = sc.model(name, C, seed=1)
    return m, sc.workload(m, 16, 200, seed=3)


def _P(w, c=0):
    return np.stack([port.expm(q) for q in w.Qt()[c]])


@pytest.mark.parametrize("name", MODELS)
def test_generators_are_not_reversible(name):
    m = sc.model(name, 3, seed=1)
    for Q in m.Q:
        pi = sc.stationary(Q)
        assert np.abs(Q.sum(axis=1)).max() <= 1e-14
        assert np.abs(pi @ Q).max() <= 1e-14 and pi.min() > 0
        flux = np.abs(pi[:, None] * Q - np.diag(pi * np.diag(Q))).max()
        assert sc.reversibility_defect(Q, pi) > 0.1 * flux, name
    if name == "drift64":
        assert np.abs(np.linalg.eigvals(m.Q[0]).imag).max() > 0.1


@pytest.mark.parametrize("name", MODELS)
def test_oracle_expm_on_nonreversible_generators(name):
    """At 1e-8, a middling length and lengths that need squarings (norm up to ~600): the oracle within the tolerance the
    GPU tests hold the engine to (a third of it), rows summing to 1."""
    Q = sc.model(name, 1, seed=1).Q[0]
    n = hc.inf_norm(Q)
    for t in (1e-8, 0.3 / n, 2.0 / n, 30.0 / n, 600.0 / n):
        A = Q * t
        P = port.expm(A)
        np.testing.assert_allclose(P, scipy.linalg.expm(A), rtol=0, atol=hc.p_atol(A) / 3, err_msg=f"{name} t={t}")
        assert np.abs(P.sum(axis=1) - 1.0).max() <= 1e-14 and P.min() >= 0


def test_nonrev_codon_template_is_the_plain_generator():
    """codon61's template assembles q_ij = rate(x -> y) * (omega if nonsynonymous), no frequencies, zero row sums."""
    m = sc.model("codon61", 2, seed=1)
    tm = m.tmpl
    assert tm.cf is None and tm.nF == 24 and len(tm.ei) == 526
    r = m.x[0].reshape(12, 2)
    Q = m.Q[0]
    i, j = np.divmod(tm.ei, 61)
    pair = tm.ef // 2
    nonsyn = tm.ef % 2
    np.testing.assert_array_equal(Q[i, j], r[pair, nonsyn])
    np.testing.assert_allclose(r[:, 1] / r[:, 0], np.full(12, 0.3))
    assert np.abs(Q.sum(axis=1)).max() <= 1e-14


@pytest.mark.parametrize("name", MODELS)
def test_oracle_pruning_at_a_nonequilibrium_root(name):
    m, w = _workload(name)
    P = _P(w, 1)
    for label, r in sc.root_vectors(w, 7).items():
        wr = sc.with_root(w, r)
        sl, ss = port.prune(wr, P)
        np.testing.assert_allclose(hc.site_lnl(sl, ss), longdouble_sites(wr, P), rtol=0, atol=1e-12, err_msg=label)


@pytest.mark.parametrize("name", MODELS)
def test_sequence_model_matches_port_lnl(name):
    """SequenceModel mixes the oracle's per-class pruning like port.lnl (same matrices, root and weights)."""
    m, w = _workload(name, C=3)
    r = sc.root_vectors(w, 2)["dirichlet"]
    sm = sc.SequenceModel(w, r, w.class_weights)
    Qt = w.Qt()
    for c in range(w.C):
        for b in range(sm.B):
            sm.set_Q(c, b, Qt[c, b])
    ref, site = port.lnl(sc.with_root(w, r), Qt, sparse_storage=False)
    got, gsite = sm.lnl()
    assert abs(got - ref) <= 1e-13 * abs(ref)
    np.testing.assert_allclose(gsite, site, rtol=0, atol=1e-12)


@pytest.mark.parametrize("name", ["nrm4", "rand20", "codon61", "drift64"])
def test_single_branch_factorisation_identity_nonreversible(name):
    """test_oracle.test_single_branch_factorisation_identity's algebra on non-reversible models at a non-equilibrium root:
    L_s = sum_a rest_b[s][a] (P_b below_b[s])[a] for every branch b, rest propagated from the root vector through the
    transposed matrices."""
    m, w = _workload(name)
    P = _P(w, 1)
    root = sc.root_vectors(w, 4)["dirichlet"]
    t = w.tree
    L, I, S = t.n_leaves, t.n_internal, w.S
    par = np.asarray(t.flat_parents)
    children = t.children()
    cond = [None] * I

    def below(n):
        if n < L:
            v = np.zeros((S, w.D))
            v[np.arange(S), w.leaf_states[n]] = 1.0
            return v
        return cond[n - L]

    for i in range(I):
        v = np.ones((S, w.D))
        for ch in children[i]:
            v *= below(ch) @ P[ch].T
        cond[i] = v
    full = cond[I - 1] @ root
    for b in range(L + I - 1):
        path, u = [], par[b]
        while u >= 0:
            path.append(u)
            u = par[L + u]
        out = np.tile(root, (S, 1))
        for k, u in enumerate(reversed(path)):
            on_path = L + path[len(path) - 2 - k] if k + 1 < len(path) else b
            rest = out.copy()
            for ch in children[u]:
                if ch != on_path:
                    rest *= below(ch) @ P[ch].T
            if k + 1 < len(path):
                out = rest @ P[on_path]
        got = np.sum(rest * (below(b) @ P[b].T), axis=1)
        assert np.abs(got / full - 1.0).max() < 1e-12, (name, b)
        if b in (0, L):            # the same with P where P^T belongs (or the reverse) is far off
            wrong = np.sum(rest * (below(b) @ P[b]), axis=1)
            assert np.abs(wrong / full - 1.0).max() > 1e-3, (name, b)


# every workload of tests/test_gpu_sequences.py: (model, classes, model seed, taxa, sites, workload seed, root-vector seed)
GPU_WORKLOADS = ([(n, 2, 1, 16, 200, 3, 3) for n in MODELS] +                        # test_nonreversible_model
                 [(n, 3, 2, 16, 150, 6, 8) for n in T.ROOTS] +                       # test_root_vector_on_every_entry_point
                 [(n, 3, s, 40, 100, s + 1, s) for n, _, s in T.SEQUENCES] +         # test_optimiser_sequence
                 [T.PLAN_CASE + (5,)])                                               # test_walk_plan_across_class_counts


@pytest.mark.parametrize("name,C,mseed,taxa,sites,wseed,rseed", GPU_WORKLOADS)
def test_rerooting_and_stationary_root_are_visible(name, C, mseed, taxa, sites, wseed, rseed):
    """The discriminating check: on every workload of the GPU tests, moving the root to a leaf or to the internal node
    farthest from it, or using the stationary vector instead of the root vector, moves lnL by at least 1e-3 relative --
    10^4 times the tensor path's tolerance; reading the longest internal branch upside down moves it by at least 1e-4."""
    m = sc.model(name, C, seed=mseed)
    w = sc.workload(m, taxa, sites, seed=wseed)
    P = _P(w, 1)
    L, I = w.tree.n_leaves, w.tree.n_internal
    r = sc.root_vectors(w, rseed)["dirichlet"]
    lnl = lambda node, root, PP=P: float((w.pattern_freq * sc.sites_rooted_at(w, PP, node, root)).sum())
    base = lnl(L + I - 1, r)
    oracle = float((w.pattern_freq * hc.site_lnl(*port.prune(sc.with_root(w, r), P))).sum())
    assert abs(base - oracle) <= 1e-13 * abs(oracle)
    deep = L + int(np.argmax(depth_of(w.tree)[L:L + I - 1]))          # the internal node farthest from the root
    long = L + int(np.argmax(w.tree.t[L:L + I - 1]))                  # the longest internal branch
    Pt = P.copy()
    Pt[long] = P[long].T
    moved = {"root at leaf 0": lnl(0, r), f"root at node {deep}": lnl(deep, r), "stationary root": lnl(L + I - 1, sc.stationary(m.Q[1])),
             f"branch {long} upside down": lnl(L + I - 1, r, Pt)}
    for label, v in moved.items():
        # one short-ish branch read upside down is a smaller change than moving the root: 1e-4, still 10^3 tolerances
        need = 1e-4 if "upside down" in label else 1e-3
        assert abs(v - base) >= need * abs(base) >= 1e3 * TC_RTOL * abs(base), (name, label, v, base)
