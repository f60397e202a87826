"""GPU suite (pytest -m gpu): the layer between the host and the kernels -- the two staging queues, compiled templates other
than id 0 with their own column frequencies, frequency changes, the shared-powers tables cached on the device across calls,
mixture groups, the tables of batched site likelihoods and the hb2_time_resident replay -- against the oracle.

Transition matrices are read back with hb2_read_transition and held to 3e-14 of the oracle's (5e-13 where the norm calls
for squarings), rows summing to 1 within 1e-14; likelihoods to the tolerances of test_gpu_parity.py.  The references are
built by tests/handover_cases.py, pinned on the CPU by tests/test_template_reference.py."""
import dataclasses

import numpy as np
import pytest

from hyphy_b200 import synth, LikelihoodFunction, engine
from oracle import port
from tests import handover_cases as hc

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
    return [(D, "fp64") for D in Ds] + [(D, "tc") for D in Ds if D > 32]


class Slots:
    """One partition and the oracle's transition matrix of every (class, branch) slot, updated with every hand-over."""

    def __init__(self, w, mode):
        self.w, self.mode = w, mode
        self.lf = LF(w, mode)
        self.part = self.lf.part
        self.B = w.tree.n_branches
        self.P = np.full((w.C, self.B, w.D, w.D), np.nan)
        self.atol = np.zeros((w.C, self.B))

    def compiled(self, tid, tmpl, c, nodes, values, shared=False):
        values = np.asarray(values, dtype=np.float64).reshape(len(nodes), tmpl.nF)
        self.part.set_matrices_compiled(c, nodes, values, template=tid)
        for b, v in zip(nodes, values):
            Q = tmpl.Q(v)
            self.P[c, b], self.atol[c, b] = hc.oracle_P(Q), hc.p_atol(Q, shared)

    def dense(self, c, nodes, Qs):
        self.part.set_matrices(c, nodes, Qs, engine.MATRIX_RATE)
        for b, Q in zip(nodes, Qs):
            self.P[c, b], self.atol[c, b] = hc.oracle_P(Q), hc.p_atol(Q)

    def trans(self, c, nodes, Ps):
        self.part.set_matrices(c, nodes, Ps, engine.MATRIX_TRANS)
        for b, P in zip(nodes, Ps):
            self.P[c, b], self.atol[c, b] = P, 0.0

    def mixture(self, c, nodes, M, wts):
        self.part.set_mixture_matrices(c, nodes, M, wts)
        for k, b in enumerate(nodes):
            self.P[c, b] = hc.mixture_P(M[k], wts[k])
            self.atol[c, b] = max(hc.p_atol(Mk) for Mk in M[k])

    def check_P(self, nodes=None, label=""):
        nodes = range(self.B) if nodes is None else nodes
        for c in range(self.w.C):
            for b in nodes:
                P = self.part.read_transition(c, b)
                err = float(np.abs(P - self.P[c, b]).max())
                assert err <= self.atol[c, b], f"{label}: class {c} branch {b}: |P - oracle| = {err:.3e} > {self.atol[c, b]:.0e}"
                rs = float(np.abs(P.sum(axis=1) - 1.0).max())
                assert rs <= 1e-14, f"{label}: class {c} branch {b}: row sums off by {rs:.3e}"

    def check_lnl(self, update_nodes=None, label=""):
        rtol, atol = tol(self.w, self.mode)
        lnl, sl, ss = self.lf.compute(update_nodes=update_nodes, want_sites=True)
        ref, site = hc.oracle_lnl(self.w, self.P)
        assert np.isfinite(lnl) and abs(lnl - ref) <= rtol * abs(ref), f"{label}: lnL {lnl!r}, oracle {ref!r}, rel {abs(lnl - ref) / abs(ref):.2e}"
        err = float(np.abs(hc.site_lnl(sl, ss) - site).max())
        assert err <= atol, f"{label}: per-pattern error {err:.2e}"
        return lnl

    def close(self):
        self.lf.close()


def report(request, case, **kv):
    """Adds measured values to the test's report (pytest --junitxml keeps them); nothing is written to the tree."""
    for k, v in kv.items():
        request.node.user_properties.append((f"{case}: {k}", repr(v)))


def model(D, C, seed):
    """Templates 0, 1, 2 and 15 of one tree: the same formulas, different column frequencies (15: none) and per-class
    formula values per unit branch length.  Returns {tid: (template, bases[C, nF])}."""
    out = {}
    for k, tid in enumerate((0, 1, 2, 15)):
        if D == 61:
            tm = hc.gy94_template(hc.codon_pi(seed + k) if k else None)
            xs = [hc.gy94_rates(2.0 + k, om) for om in np.linspace(0.2, 1.6, C) * (1 + 0.3 * k)]
        else:
            tm, x = hc.gtr_template(D, seed + k)
            xs = [x * (1.0 + 0.5 * c) * np.random.default_rng(seed + 10 * k + c).uniform(0.7, 1.3, x.size) for c in range(C)]
        if tid == 15:
            tm = tm.with_freqs(None)
        out[tid] = (tm, np.stack([hc.unit_rate(tm, x) for x in xs]))
    return out


def values(base, t, nodes, scale=1.0):
    return base[None, :] * (np.asarray(t)[nodes] * scale)[:, None]


# ---------------------------------------------------------------------------------------------------------------------
# 1. several templates on one tree
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D,mode", with_modes([61, 48, 20]))
def test_several_templates_on_one_tree(D, mode):
    """Template 0 on most branches, template 1 on 28 (a shared-powers group of its own), template 2 on 3, template 15 -- the
    highest id, no column frequencies -- on 1: every matrix and the likelihood follow their own template."""
    w = hc.workload(D, 40, 120, 2, mean_t=0.1)
    h = Slots(w, mode)
    t = w.tree.t
    m = model(D, 2, 100 + D)
    assign = {2: [0, 1, 2], 15: [3], 1: list(range(4, 32)), 0: list(range(32, h.B))}
    for tid, (tm, _) in m.items():
        tm.define(h.part, tid)
    for tid, nodes in assign.items():
        tm, base = m[tid]
        for c in range(w.C):
            h.compiled(tid, tm, c, nodes, values(base[c], t, nodes))
    h.check_lnl(label="templates 0, 1, 2, 15")
    h.check_P(label="templates 0, 1, 2, 15")
    h.close()


# ---------------------------------------------------------------------------------------------------------------------
# 2. frequency changes
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", list(MODES))
def test_frequency_changes(mode):
    """(a) new frequencies and every branch handed over again; (c) new frequencies and nothing handed over: the resident
    matrices do not move; (b) new frequencies, then one branch proportional to the last reference of its shared-powers group
    and one that is not: both follow the new frequencies."""
    w = hc.workload(61, 40, 120, 2, mean_t=0.1)
    h = Slots(w, mode)
    t, nodes = w.tree.t, np.arange(h.B)
    tm = hc.gy94_template()
    tm.define(h.part, 0)
    bases = [hc.unit_rate(tm, hc.gy94_rates(2.0, om)) for om in (0.2, 1.5)]

    def all_over(tm):
        for c in range(w.C):
            h.compiled(0, tm, c, nodes, values(bases[c], t, nodes))

    all_over(tm)
    h.check_lnl(label="start")
    h.check_P(label="start")
    tm = tm.with_freqs(hc.codon_pi(11))                         # (a)
    h.part.set_template_frequencies(0, tm.cf)
    all_over(tm)
    h.check_lnl(label="(a) all handed over again")
    h.check_P(label="(a) all handed over again")
    before = h.lf.compute()                                     # (c)
    tm = tm.with_freqs(hc.codon_pi(12))
    h.part.set_template_frequencies(0, tm.cf)
    after = h.lf.compute()
    assert after == before, f"(c) a frequency change alone moved the lnL: {before!r} -> {after!r}"
    h.check_P(label="(c) nothing handed over")
    other = hc.unit_rate(tm, hc.gy94_rates(3.0, 0.7))          # (b)
    for c in range(w.C):
        h.compiled(0, tm, c, [7], values(bases[c], t, [7], 1.75))
        h.compiled(0, tm, c, [9], values(other, t, [9]))
    h.check_P([7, 9], label="(b) proportional branch 7, other branch 9 after a frequency change")
    h.check_lnl(update_nodes=[7, 9], label="(b)")
    h.close()


def test_frequency_change_error_paths():
    w = hc.workload(61, 8, 20, 1)
    lf = LF(w, "fp64")
    tm = hc.gy94_template()
    lf.part.set_rate_template_id(0, tm.ei, tm.ef, tm.nF, None)
    with pytest.raises(engine.EngineError, match="without column frequencies"):
        lf.part.set_template_frequencies(0, tm.cf)
    for tid in (3, 15, 16):
        with pytest.raises(engine.EngineError, match="has not been defined"):
            lf.part.set_template_frequencies(tid, tm.cf)
    with pytest.raises(engine.EngineError, match="template 3"):
        lf.part.set_matrices_compiled(0, [0], np.ones((1, tm.nF)), template=3)
    lf.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3. template redefinition
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", list(MODES))
def test_template_redefinition_uses_the_new_scatter(mode):
    """Template 0 redefined with the same formula count and a permuted formula map; a branch then handed over with values
    proportional to the old reference direction is assembled with the new map."""
    w = hc.workload(61, 40, 120, 1, mean_t=0.1)
    h = Slots(w, mode)
    t, nodes = w.tree.t, np.arange(h.B)
    tm = hc.gy94_template()
    tm.define(h.part, 0)
    base = hc.unit_rate(tm, hc.gy94_rates(2.5, 0.3))
    h.compiled(0, tm, 0, nodes, values(base, t, nodes))
    h.check_lnl(label="before")
    tm2 = dataclasses.replace(tm, ef=np.array([2, 3, 0, 1])[tm.ef])
    tm2.define(h.part, 0)
    h.compiled(0, tm2, 0, [5], values(base, t, [5], 1.3))
    h.check_P(label="after redefinition")
    h.check_lnl(update_nodes=[5], label="after redefinition")
    h.close()


# ---------------------------------------------------------------------------------------------------------------------
# 4. template groups and mixture groups that share an index
# ---------------------------------------------------------------------------------------------------------------------
def mixture_inputs(tm, t, nodes, scale=1.0, omegas=(0.1, 1.0, 4.0), wts=(0.6, 0.3, 0.1)):
    Qk = [tm.Q(hc.unit_rate(tm, hc.gy94_rates(2.0, om))) for om in omegas]
    M = np.stack([np.stack([Q * (t[b] * scale) for Q in Qk]) for b in nodes])
    return M, np.tile(np.asarray(wts, dtype=np.float64), (len(nodes), 1))


@pytest.mark.parametrize("C,mode", [(1, "fp64"), (1, "tc"), (4, "fp64"), (4, "tc")])
def test_template_and_mixture_groups_sharing_an_index(C, mode):
    """Template 1's shared-powers groups (1 * C + class) and mixture component k's (C + k) coincide: a table built for one
    must never serve the other."""
    w = hc.workload(61, 40, 100, C, mean_t=0.1)
    h = Slots(w, mode)
    t = w.tree.t
    A, M, R = np.arange(0, 30), np.arange(30, 60), np.arange(60, h.B)
    t0, t1 = hc.gy94_template(), hc.gy94_template(hc.codon_pi(21))
    t0.define(h.part, 0)
    t1.define(h.part, 1)
    om = np.linspace(0.3, 1.2, C)
    b0 = [hc.unit_rate(t0, hc.gy94_rates(2.0, o)) for o in om]
    b1 = [hc.unit_rate(t1, hc.gy94_rates(3.0, 2 * o)) for o in om]
    for c in range(C):
        h.compiled(1, t1, c, A, values(b1[c], t, A))
        h.compiled(0, t0, c, np.r_[M, R], values(b0[c], t, np.r_[M, R]))
    h.check_lnl(label="1: template 1 on 30 branches")
    h.check_P(label="1: template 1 on 30 branches")
    for c in range(C):
        h.mixture(c, M, *mixture_inputs(t0, t, M, 1.0 + 0.2 * c))
    h.check_lnl(label="2: mixture on 30 branches")
    h.check_P(label="2: mixture on 30 branches")
    for c in range(C):
        h.compiled(1, t1, c, [3], values(b1[c], t, [3], 1.4))
    h.check_P(label="3: one proportional template-1 branch")
    h.check_lnl(update_nodes=[3], label="3: one proportional template-1 branch")
    for c in range(C):
        h.mixture(c, [31, 32], *mixture_inputs(t0, t, [31, 32], 1.2 * (1.0 + 0.2 * c)))
    h.check_P(label="4: mixture on 2 proportional branches")
    h.check_lnl(update_nodes=[31, 32], label="4: mixture on 2 proportional branches")
    h.close()


# ---------------------------------------------------------------------------------------------------------------------
# 5. one slot changes kind across evaluations
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", list(MODES))
def test_slots_change_kind_across_evaluations(mode):
    """The same branches go compiled (template 0) -> compiled (template 1) -> dense rate matrix -> transition matrix ->
    mixture -> compiled (template 0), with a partial evaluation after each step; fp64: equal to a full one bit for bit."""
    w = hc.workload(61, 40, 100, 2, mean_t=0.1)
    h = Slots(w, mode)
    t, L = w.tree.t, w.tree.n_leaves
    S = [2, 11, L + 4]
    t0, t1 = hc.gy94_template(), hc.gy94_template(hc.codon_pi(31))
    t0.define(h.part, 0)
    t1.define(h.part, 1)
    b0 = [hc.unit_rate(t0, hc.gy94_rates(2.0, o)) for o in (0.3, 1.1)]
    b1 = [hc.unit_rate(t1, hc.gy94_rates(4.0, o)) for o in (0.5, 2.0)]
    nodes = np.arange(h.B)
    for c in range(w.C):
        h.compiled(0, t0, c, nodes, values(b0[c], t, nodes))
    h.check_lnl(label="start")
    dense = [t0.Q(hc.unit_rate(t0, hc.gy94_rates(1.5, o))) for o in (0.2, 0.9)]
    steps = [
        ("template 0", lambda c: h.compiled(0, t0, c, S, values(b0[c], t, S, 1.1))),
        ("template 1", lambda c: h.compiled(1, t1, c, S, values(b1[c], t, S))),
        ("dense rate matrix", lambda c: h.dense(c, S, np.stack([dense[c] * t[b] for b in S]))),
        ("transition matrix", lambda c: h.trans(c, S, np.stack([hc.oracle_P(dense[c] * (1.3 * t[b])) for b in S]))),
        ("mixture", lambda c: h.mixture(c, S, *mixture_inputs(t0, t, S, 0.8 + 0.4 * c))),
        ("template 0 again", lambda c: h.compiled(0, t0, c, S, values(b0[c], t, S, 0.9))),
    ]
    for label, step in steps:
        for c in range(w.C):
            step(c)
        h.check_P(S, label=label)
        part = h.check_lnl(update_nodes=S, label=label)
        full = h.lf.compute()
        if mode == "fp64":
            assert part == full, f"{label}: partial {part!r} != full {full!r}"
        else:
            assert abs(part - full) <= 1e-9 * abs(full), f"{label}: partial {part!r}, full {full!r}"
    h.close()


# ---------------------------------------------------------------------------------------------------------------------
# 6. queue overflow before an evaluation
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("first", ["dense", "compiled"])
@pytest.mark.parametrize("mode", list(MODES))
def test_queue_overflow_before_an_evaluation(first, mode):
    """Every slot handed over twice in one form and every other slot once in the other in between, with no evaluation: the
    queues (one matrix per slot each) overflow with live entries in both and flush mid-queue.  The last hand-over wins."""
    w = hc.workload(61, 40, 100, 2, mean_t=0.1)
    h = Slots(w, mode)
    t = w.tree.t
    tm = hc.gy94_template()
    tm.define(h.part, 0)
    all_, even = np.arange(h.B), np.arange(0, h.B, 2)

    def hand(kind, nodes, kappa, omega, scale):
        for c in range(w.C):
            base = hc.unit_rate(tm, hc.gy94_rates(kappa, omega * (1 + c)))
            if kind == "compiled":
                h.compiled(0, tm, c, nodes, values(base, t, nodes, scale))
            else:
                h.dense(c, nodes, np.stack([tm.Q(base) * (t[b] * scale) for b in nodes]))

    other = "compiled" if first == "dense" else "dense"
    hand(first, all_, 2.0, 0.3, 1.0)
    hand(other, even, 3.0, 0.6, 1.25)
    hand(first, all_, 1.5, 0.2, 0.8)
    h.check_lnl(label=f"{first}/{other}/{first}")
    h.check_P(label=f"{first}/{other}/{first}")
    h.close()


# ---------------------------------------------------------------------------------------------------------------------
# 7. the proportionality tolerance and the polynomial's range, with column frequencies
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", list(MODES))
def test_proportionality_tolerance_and_polynomial_range(mode):
    """Single branches handed over with values equal to the group's reference times c, up to relative noise of 1e-15,
    1e-13 * (1 +- 0.5) and 1e-11 on one formula: within 3e-14 of the oracle on whichever path the engine takes.  Then
    proportional branches whose norm lies just below and just above EXPM_POLY_THETA."""
    w = hc.workload(61, 40, 100, 1, mean_t=0.1)
    h = Slots(w, mode)
    t, nodes = w.tree.t, np.arange(h.B)
    tm = hc.gy94_template()
    tm.define(h.part, 0)
    base = hc.unit_rate(tm, hc.gy94_rates(2.0, 0.4))
    h.compiled(0, tm, 0, nodes, values(base, t, nodes))
    h.check_lnl(label="start")
    rng = np.random.default_rng(7)
    b, rho = 6, hc.inf_norm(tm.Q(base))
    v = base * (0.3 / rho)                                     # norm 0.3
    cases = [("noise 1e-15", v * (1 + 1e-15 * rng.uniform(-1, 1, v.size))),
             ("noise 1e-13*(1+-0.5)", v * (1 + 1e-13 * rng.choice([-1.0, 1.0], v.size) * rng.uniform(0.5, 1.5, v.size))),
             ("1e-11 on one formula", v * np.where(np.arange(v.size) == 1, 1 + 1e-11, 1.0))]
    for label, vv in cases:
        h.compiled(0, tm, 0, [b], vv[None])
        assert h.atol[0, b] == 3e-14
        h.check_P([b], label=label)
    for target in (2.29, 2.31):
        h.compiled(0, tm, 0, [b], (base * (target / rho))[None], shared=True)
        h.check_P([b], label=f"norm {target}")
    h.check_lnl(update_nodes=[b], label="end")
    h.close()


# ---------------------------------------------------------------------------------------------------------------------
# 8. hb2_time_resident
# ---------------------------------------------------------------------------------------------------------------------
RESIDENT_RTOL = {"fp64": 1e-12, "tc": 1e-9}


def _resident_case(case):
    if case == "d4":
        return synth.nucleotide_workload(64, 2000, mean_t=0.1)
    if case == "d20":
        return synth.generic_workload(20, 32, 2000, 4, mean_t=0.1)
    return synth.codon_workload(40, 300, 4, mean_t=0.1)


@pytest.mark.parametrize("case,mode", [(c, m) for c in ("dense", "compiled", "compiled+partial") for m in MODES] +
                         [("d4", "fp64"), ("d20", "fp64")])
def test_time_resident_matches_compute(case, mode, request):
    """The replay behind bench.py's `value`: its lnL equals compute()'s on the same resident matrices."""
    w = _resident_case(case)
    lf = LF(w, mode)
    lf.set_template()
    lf.set_all_compiled()
    Qt = w.Qt()
    first = lf.compute()
    if case == "dense":
        for c in range(w.C):
            lf.part.set_matrices(c, lf.all_nodes, Qt[c])
    lf.part.time_resident(w.class_weights, w.pi, iters=2)
    if case == "compiled+partial":
        b = 5
        Qt[:, b] *= 1.3
        V = w.compiled_values()
        for c in range(w.C):
            lf.part.set_matrices_compiled(c, [b], V[c, b:b + 1] * 1.3)
        lf.compute(update_nodes=[b])
    _, _, res = lf.part.time_resident(w.class_weights, w.pi, iters=2)
    lnl = lf.compute()
    lf.close()
    ref = port.lnl(w, Qt)[0]
    report(request, case, resident=res, compute=lnl, first=first, oracle=ref, bit_identical=res == lnl)
    assert abs(res - lnl) <= RESIDENT_RTOL[mode] * abs(lnl), f"{case}: resident {res!r}, compute {lnl!r}"
    assert abs(lnl - ref) <= tol(w, mode)[0] * abs(ref), f"{case}: compute {lnl!r}, oracle {ref!r}"


@pytest.mark.parametrize("mode", list(MODES))
def test_time_resident_refuses_what_it_cannot_replay(mode, request):
    """A mixture slot, a template-1 slot and a frequency change with nothing handed over again make the replay fail with a
    message (it would time a different model than the last evaluation); after a full hand-over it agrees again."""
    w = hc.workload(61, 40, 100, 1, mean_t=0.1)
    lf = LF(w, mode)
    p = lf.part
    t, nodes = w.tree.t, lf.all_nodes
    t0, t1 = hc.gy94_template(), hc.gy94_template(hc.codon_pi(51))
    t0.define(p, 0)
    t1.define(p, 1)
    base = hc.unit_rate(t0, hc.gy94_rates(2.0, 0.5))
    wts = np.ones(1)

    def agrees(label):
        lnl = p.evaluate_classes(wts, w.pi)
        _, _, res = p.time_resident(wts, w.pi, iters=1)
        report(request, label, resident=res, compute=lnl, bit_identical=res == lnl)
        assert abs(res - lnl) <= RESIDENT_RTOL[mode] * abs(lnl), f"{label}: resident {res!r}, compute {lnl!r}"

    p.set_matrices_compiled(0, nodes, values(base, t, nodes))
    agrees("template 0 with column frequencies")
    p.set_mixture_matrices(0, [4], *mixture_inputs(t0, t, [4]))
    p.evaluate_classes(wts, w.pi)
    with pytest.raises(engine.EngineError, match="hb2_time_resident"):
        p.time_resident(wts, w.pi, iters=1)
    p.set_matrices_compiled(0, [4], values(base, t, [4]))
    agrees("mixture replaced")
    p.set_matrices_compiled(0, [4], values(base, t, [4]), template=1)
    p.evaluate_classes(wts, w.pi)
    with pytest.raises(engine.EngineError, match="hb2_time_resident"):
        p.time_resident(wts, w.pi, iters=1)
    p.set_matrices_compiled(0, [4], values(base, t, [4]))
    agrees("template-1 slot replaced")
    p.set_template_frequencies(0, hc.codon_pi(52))
    with pytest.raises(engine.EngineError, match="hb2_time_resident"):
        p.time_resident(wts, w.pi, iters=1)
    p.set_matrices_compiled(0, nodes, values(base, t, nodes))
    agrees("all handed over after the frequency change")
    lf.close()


# ---------------------------------------------------------------------------------------------------------------------
# 9. batched site likelihoods
# ---------------------------------------------------------------------------------------------------------------------
def test_batched_site_likelihoods_follow_template_and_frequencies():
    """Calls alternate between two branch-group layouts -- in one, groups 1..3 have 4 or more branches (their power tables
    are built), in the other 1, 2 and 3 (they are compared with a cached direction) -- and between templates 0 and 1, which
    have the same formulas and different column frequencies, with a frequency change in between.  1100 sets: two chunks."""
    w = hc.workload(61, 16, 60, 1, mean_t=0.1)
    lf = LF(w, "fp64")
    p = lf.part
    B, t = w.tree.n_branches, w.tree.t
    tms = {0: hc.gy94_template(), 1: hc.gy94_template(hc.codon_pi(61))}
    for tid, tm in tms.items():
        tm.define(p, tid)
    big = np.zeros(B, dtype=np.int64)                     # groups 0: 8 branches, 1: 4, 2: 4, 3: 13
    big[8:12], big[12:16], big[16:] = 1, 2, 3
    small = np.zeros(B, dtype=np.int64)                   # groups 1: 1 branch, 2: 2, 3: 3, 0: the other 23
    small[8], small[12:14], small[16:19] = 1, 2, 3
    nSets = 1100
    rng = np.random.default_rng(5)
    omega = rng.uniform(0.05, 3.0, size=(nSets, 4))       # per set and (big-layout) branch group
    scale = hc.unit_rate(tms[0], hc.gy94_rates(2.0, 1.0))[0]
    V = np.stack([np.stack([hc.gy94_rates(2.0, omega[s, big[b]]) * scale * t[b] for b in range(B)]) for s in range(nSets)])
    pattern_of = np.arange(nSets) % w.S
    sample = sorted(set(range(0, nSets, 37)) | {0, 1023, 1024, nSets - 1})
    refs = {}

    def call(tid, layout, label):
        tm = tms[tid]
        out = p.batch_site_likelihoods(pattern_of, V, w.pi, layout, template=tid)
        key = tm.cf.tobytes()
        for s in sample:
            if (key, s) not in refs:
                P = np.stack([hc.oracle_P(tm.Q(V[s, b])) for b in range(B)])
                refs[key, s] = hc.site_lnl(*port.prune(w, P))[pattern_of[s]]
            ref = refs[key, s]
            assert abs(out[s] - ref) <= 1e-10 * abs(ref), f"{label}: set {s} (chunk {s // 1024}): {out[s]!r}, oracle {ref!r}"

    call(0, big, "template 0, groups of 4+")
    call(1, small, "template 1, groups of 1-3")
    call(1, big, "template 1, groups of 4+")
    tms[0] = tms[0].with_freqs(hc.codon_pi(62))
    p.set_template_frequencies(0, tms[0].cf)
    call(0, small, "template 0 after a frequency change, groups of 1-3")
    call(0, big, "template 0 after a frequency change, groups of 4+")
    lf.close()


# ---------------------------------------------------------------------------------------------------------------------
# 10. refused hand-overs
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("form", ["dense", "compiled template 0", "compiled template 1", "mixture"])
def test_refused_handovers_change_nothing(form):
    """A hand-over whose last node id is B (no such branch) is refused as a whole.  (a) On a fresh partition in which every
    other slot holds a matrix, the listed slots still hold none: compute() fails with "no matrix was ever set".  (b) On an
    evaluated partition, the listed valid slots keep their matrices bit for bit, a branch cache built before the call still
    evaluates, and a re-evaluation gives the same lnL bit for bit."""
    w = hc.workload(61, 12, 40, 2, mean_t=0.1)
    t = w.tree.t
    tm = hc.gy94_template()
    base = hc.unit_rate(tm, hc.gy94_rates(2.0, 0.5))
    c, listed = 1, np.array([2, 7])
    refused = np.r_[listed, w.tree.n_branches]

    def fresh():
        lf = LF(w, "fp64")
        tm.define(lf.part, 0)
        tm.with_freqs(hc.codon_pi(71)).define(lf.part, 1)
        return lf

    def refuse(part):
        v = values(base, t, refused % w.tree.n_branches, 1.3)
        with pytest.raises(engine.EngineError, match="has no branch"):
            if form == "dense":
                part.set_matrices(c, refused, np.stack([tm.Q(x) for x in v]), engine.MATRIX_RATE)
            elif form == "mixture":
                part.set_mixture_matrices(c, refused, *mixture_inputs(tm, t, refused % w.tree.n_branches, 1.3))
            else:
                part.set_matrices_compiled(c, refused, v, template=int(form[-1]))

    lf = fresh()                                                                         # (a)
    nodes = lf.all_nodes
    for cc in range(w.C):
        rest = nodes if cc != c else np.setdiff1d(nodes, listed)
        lf.part.set_matrices_compiled(cc, rest, values(base, t, rest))
    refuse(lf.part)
    with pytest.raises(engine.EngineError, match="no matrix was ever set"):
        lf.compute()
    lf.close()

    lf = fresh()                                                                         # (b)
    for cc in range(w.C):
        lf.part.set_matrices_compiled(cc, nodes, values(base, t, nodes))
    before = lf.compute()
    P = [lf.part.read_transition(c, b) for b in listed]
    lf.part.branch_cache_build(int(listed[0]), w.pi)
    refuse(lf.part)
    cached = lf.part.branch_cache_evaluate(w.class_weights)
    assert abs(cached - before) <= 1e-10 * abs(before), f"branch cache {cached!r}, full {before!r}"
    for b, Pb in zip(listed, P):
        assert np.array_equal(lf.part.read_transition(c, b), Pb), f"{form}: the matrix of branch {b} changed"
    after = lf.compute()
    assert after == before, f"{form}: lnL {before!r} -> {after!r}"
    lf.close()
