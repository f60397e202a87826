"""Reference builders for the non-reversible and sequence tests: non-reversible generators with their stationary vectors,
workloads simulated under them, root vectors other than the stationary one, a numpy likelihood that can put the root at
any node, and `SequenceModel`, which holds what a partition should hold after any sequence of hand-overs and computes the
oracle's likelihoods from scratch.  No test functions live here."""
import dataclasses

import numpy as np
import scipy.linalg

from hyphy_b200 import synth
from oracle import port
from tests import handover_cases as hc


# ---------------------------------------------------------------------------------------------------------------------
# generators
# ---------------------------------------------------------------------------------------------------------------------
def stationary(Q):
    """pi with pi Q = 0 and sum(pi) = 1 (least squares on the stacked system)."""
    D = Q.shape[0]
    A = np.vstack([Q.T, np.ones((1, D))])
    b = np.zeros(D + 1)
    b[-1] = 1.0
    pi = np.linalg.lstsq(A, b, rcond=None)[0]
    return pi / pi.sum()


def from_rates(R):
    """Generator with off-diagonal rates R, zero row sums, scaled to one expected substitution per unit length under its
    stationary vector.  Returns (Q, pi)."""
    Q = np.array(R, dtype=np.float64)
    Q[np.diag_indices(Q.shape[0])] = 0.0
    Q[np.diag_indices(Q.shape[0])] = -Q.sum(axis=1)
    pi = stationary(Q)
    return Q / -(pi * np.diag(Q)).sum(), pi


def nrm_Q(seed):
    """4 states, NRM shape: 12 free rates."""
    return from_rates(np.random.default_rng(seed).gamma(1.0, 1.0, size=(4, 4)))


def random_Q(D, seed):
    """D states, every off-diagonal rate drawn independently."""
    return from_rates(np.random.default_rng(seed).gamma(0.7, 1.0, size=(D, D)))


def drift_Q(D, seed, forward=1.0, backward=0.02, noise=0.002):
    """A cyclic drift i -> i+1 (mod D) at a large rate and back at a small one, plus weak uniform noise: strongly
    non-normal, with complex eigenvalues."""
    rng = np.random.default_rng(seed)
    R = noise * rng.uniform(0.5, 1.5, size=(D, D))
    i = np.arange(D)
    R[i, (i + 1) % D] += forward * rng.uniform(0.8, 1.2, D)
    R[i, (i - 1) % D] += backward * rng.uniform(0.8, 1.2, D)
    return from_rates(R)


def nonrev_codon_template():
    """61 sense codons, MG94 shape with a non-reversible nucleotide part and no column frequencies (the "do not multiply
    by frequencies" form): one formula per (ordered nucleotide pair, nonsynonymous), formula 2 * pair + nonsynonymous
    with the 12 ordered pairs numbered row by row."""
    pairs = [(x, y) for x in range(4) for y in range(4) if x != y]
    pid = {p: k for k, p in enumerate(pairs)}
    ei, ef = [], []
    for i, ci in enumerate(synth.SENSE):
        for shift in (4, 2, 0):
            x = (ci >> shift) & 3
            for y in range(4):
                cj = (ci & ~(3 << shift)) | (y << shift)
                if y == x or cj in synth.STOPS:
                    continue
                ei.append(i * 61 + synth.SENSE_INDEX[cj])
                ef.append(2 * pid[x, y] + int(synth._AA[ci] != synth._AA[cj]))
    return hc.Template(np.array(ei, dtype=np.int64), np.array(ef, dtype=np.int64), 24, None, 61)


def codon_rates(seed, omega):
    """Formula values of nonrev_codon_template: 12 random ordered nucleotide rates, times omega where nonsynonymous."""
    r = np.random.default_rng(seed).gamma(1.0, 1.0, size=12)
    return np.stack([r, r * omega], axis=1).reshape(-1)


def generic_template(D):
    """Every off-diagonal entry its own formula, no column frequencies."""
    ei = np.array([i * D + j for i in range(D) for j in range(D) if i != j], dtype=np.int64)
    return hc.Template(ei, np.arange(len(ei), dtype=np.int64), len(ei), None, D)


def offdiag(Q):
    D = Q.shape[0]
    return np.array([Q[i, j] for i in range(D) for j in range(D) if i != j])


@dataclasses.dataclass
class Model:
    """Per-class generators with the compiled form that gives them: Q[c] = template.Q(x[c])."""
    name: str
    tmpl: hc.Template
    x: np.ndarray               # [C, nF] formula values per unit length
    Q: np.ndarray               # [C, D, D]
    pi: np.ndarray              # stationary vector of class 0

    @property
    def D(self):
        return self.tmpl.D


def model(name, C=1, seed=0):
    """Non-reversible models: nrm4, rand8, rand20, rand24, codon61 (MG94 shape, non-reversible, no frequencies), drift64.
    Classes differ by rate (generic templates) or by omega (codon61)."""
    if name == "codon61":
        tm = nonrev_codon_template()
        xs = [codon_rates(seed, om) for om in np.linspace(0.3, 1.5, C)]
        Q0 = tm.Q(xs[0])
        sc = -(stationary(Q0) * np.diag(Q0)).sum()
        xs = [x / sc for x in xs]
    else:
        kind = name.rstrip("0123456789")
        D = int(name[len(kind):])
        Q0, _ = {"nrm": lambda: nrm_Q(seed), "rand": lambda: random_Q(D, seed + D), "drift": lambda: drift_Q(D, seed + D)}[kind]()
        tm = generic_template(D)
        xs = [offdiag(Q0) * r for r in np.linspace(1.0, 2.0, C) / np.linspace(1.0, 2.0, C).mean()]
    Q = np.stack([tm.Q(x) for x in xs])
    return Model(name, tm, np.stack(xs), Q, stationary(Q[0]))


def reversibility_defect(Q, pi):
    """max |pi_i Q_ij - pi_j Q_ji|: 0 for a reversible generator."""
    F = pi[:, None] * Q
    return float(np.abs(F - F.T).max())


# ---------------------------------------------------------------------------------------------------------------------
# workloads and root vectors
# ---------------------------------------------------------------------------------------------------------------------
def workload(m, n_taxa, n_sites, seed=5, mean_t=0.15, weights=None):
    """An alignment simulated under class 0 of model m (root states drawn from its stationary vector) on a random tree;
    the workload's Q_classes are m's, its pi the stationary vector."""
    rng = np.random.default_rng(seed)
    tree = synth.random_tree(n_taxa, seed + n_taxa, mean_t)
    nb = tree.n_branches
    Ps = [[scipy.linalg.expm(m.Q[0] * tree.t[b]) for b in range(nb)]]
    states = synth._simulate(tree, Ps, m.pi, np.zeros(n_sites, dtype=np.int64), rng)
    ls, freq, s2p = synth.compress(states)
    C = m.Q.shape[0]
    cw = np.linspace(1.0, 2.0, C) if weights is None else np.asarray(weights, dtype=np.float64)
    return synth.Workload(f"{m.name}_{n_taxa}x{n_sites}", tree, m.D, m.pi.copy(), list(m.Q), cw / cw.sum(), ls,
                          np.zeros((0, m.D)), freq, s2p, None, {"kind": "nonrev"})


def with_root(w, root):
    """A copy of workload w whose pi -- the vector the oracle's pruning puts at the root -- is `root`."""
    return dataclasses.replace(w, pi=np.asarray(root, dtype=np.float64).copy())


def root_vectors(w, seed):
    """Root vectors other than the stationary one: a random Dirichlet vector, one with zeros in a third of the states,
    and a point mass on the state the leaves show most often (every pattern stays possible: all P entries are positive)."""
    rng = np.random.default_rng(seed)
    D = w.D
    dirichlet = rng.dirichlet(np.full(D, 1.0))
    zeros = rng.dirichlet(np.full(D, 1.0))
    zeros[rng.choice(D, size=D // 3, replace=False)] = 0.0
    zeros /= zeros.sum()
    point = np.zeros(D)
    point[np.bincount(w.leaf_states[w.leaf_states >= 0], minlength=D).argmax()] = 1.0
    return {"dirichlet": dirichlet, "zeros": zeros, "point": point}


def oracle_P(Q):
    return port.expm(Q)


# ---------------------------------------------------------------------------------------------------------------------
# a likelihood with the root at any node
# ---------------------------------------------------------------------------------------------------------------------
def sites_rooted_at(w, P, root_node, root):
    """Per-pattern log-likelihoods with the root vector at node `root_node` (flat id) and every branch b (named by its
    child in w's flat layout) read with its matrix P[b] from whichever end is nearer the new root: P[b][a_near][a_far].
    At w's own root this is Felsenstein's recursion on w; elsewhere it is w re-rooted."""
    L, I = w.tree.n_leaves, w.tree.n_internal
    par = np.asarray(w.tree.flat_parents)
    adj = [[] for _ in range(L + I)]                      # (neighbour, branch id)
    for n in range(L + I - 1):
        adj[n].append((L + par[n], n))
        adj[L + par[n]].append((n, n))
    order, parent_of, stack = [], {root_node: (-1, -1)}, [root_node]
    while stack:
        u = stack.pop()
        order.append(u)
        for v, b in adj[u]:
            if v not in parent_of:
                parent_of[v] = (u, b)
                stack.append(v)
    vec, logs = {}, {}
    for u in reversed(order):                             # children before parents
        if u < L:
            v = np.zeros((w.S, w.D))
            v[np.arange(w.S), w.leaf_states[u]] = 1.0
            lg = np.zeros(w.S)
        else:
            v, lg = np.ones((w.S, w.D)), np.zeros(w.S)
        for c, b in adj[u]:
            if parent_of.get(c, (None,))[0] == u:
                v = v * (vec[c] @ P[b].T)
                lg = lg + logs[c]
                m = v.max(axis=1, keepdims=True)
                v, lg = v / m, lg + np.log(m[:, 0])
        vec[u], logs[u] = v, lg
    return np.log(vec[root_node] @ root) + logs[root_node]


# ---------------------------------------------------------------------------------------------------------------------
# what a partition should hold
# ---------------------------------------------------------------------------------------------------------------------
class SequenceModel:
    """The dense transition matrix of every (class, branch) slot, the root vector and the class weights, as a partition
    should hold them after a sequence of hand-overs; oracle likelihoods from scratch on demand, with the per-class pruning
    cached until that class's matrices or the root vector change."""

    def __init__(self, w, root, weights):
        self.w = w
        self.B = w.tree.n_branches
        self.P = np.full((w.C, self.B, w.D, w.D), np.nan)
        self.atol = np.zeros((w.C, self.B))
        self.root = np.asarray(root, dtype=np.float64).copy()
        self.weights = np.asarray(weights, dtype=np.float64).copy()
        self._sites = {}

    def set_P(self, c, b, P, atol=0.0):
        self.P[c, b], self.atol[c, b] = P, atol
        self._sites.pop(c, None)

    def set_Q(self, c, b, Q, shared_powers=False):
        self.set_P(c, b, oracle_P(Q), hc.p_atol(Q, shared_powers))

    def set_mixture(self, c, b, Ms, wts):
        self.set_P(c, b, hc.mixture_P(Ms, wts), max(hc.p_atol(M) for M in Ms))

    def set_root(self, root):
        self.root = np.asarray(root, dtype=np.float64).copy()
        self._sites.clear()

    def rooted(self):
        return with_root(self.w, self.root)

    def class_sites(self, c):
        """Per-pattern log-likelihoods of class c."""
        if c not in self._sites:
            self._sites[c] = hc.site_lnl(*port.prune(self.rooted(), self.P[c]))
        return self._sites[c]

    def class_lnl(self, c):
        s = self.class_sites(c)
        return float((self.w.pattern_freq * s).sum()), s

    def lnl(self, weights=None):
        """(lnL, per-pattern values) mixed over the classes."""
        wts = self.weights if weights is None else weights
        sites = np.stack([self.class_sites(c) for c in range(self.w.C)])
        m = sites.max(axis=0)
        site = m + np.log(np.einsum("c,cs->s", wts, np.exp(sites - m)))
        return float((self.w.pattern_freq * site).sum()), site

    def forced_sites(self, c, node, states):
        sl, ss = port.prune_forced(self.rooted(), self.P[c], node, states)
        return hc.site_lnl(np.maximum(sl, 1e-300), ss), sl > 0

    def conditionals(self, c):
        """The oracle's conditionals of class c [I, S, D] (a row multiplied by 2^64 whenever it fell below 2^-64)."""
        return port.prune(self.rooted(), self.P[c], want_cond=True)[2]
