"""numpy restatement of hb2_batch_site_simulate's stream (include/hyphy_b200.h): hb2_simulate's Philox4x32-10, uniform and
draw rule (tests/simulate_reference.py) with the global set t in the fourth counter word and no class draw.  Fed the
engine's own per-set matrices it must reproduce the engine's output bit for bit.  No test functions live here."""
import numpy as np

from tests.simulate_reference import philox4x32_10, prefix, draw

_MASK = np.uint64(0xFFFFFFFF)


def uniforms(g, slot, t, seed):
    """u of draw `slot` for global replicates g and global sets t (arrays, broadcast against each other)."""
    g, t = np.broadcast_arrays(np.asarray(g, dtype=np.uint64), np.asarray(t, dtype=np.uint64))
    seed = np.uint64(seed)
    ctr = np.stack([g & _MASK, g >> np.uint64(32), np.full_like(g, slot), t & _MASK], axis=-1)
    key = np.array([seed & _MASK, seed >> np.uint64(32)], dtype=np.uint64)
    x = philox4x32_10(ctr, key).astype(np.uint64)
    return ((x[..., 0] << np.uint64(21)) + (x[..., 1] >> np.uint64(11))).astype(np.float64) * 2.0 ** -53


def mix(P, weights, branch_k):
    """Per-branch matrices [B, D, D] of one set from its component matrices [R, D, D] and weights [R], components of a
    branch consecutive and added in order."""
    out, r = [], 0
    for k in branch_k:
        acc = weights[r] * P[r]
        for c in range(1, k):
            acc = acc + weights[r + c] * P[r + c]
        out.append(acc)
        r += k
    return np.stack(out)


def simulate_sets(P, root_freqs, flat_parents, n_leaves, n_reps, seed, first_set=0, first_rep=0):
    """P [nSets, B, D, D] (row = parent state): each set's own matrices.  Returns (leaf [nSets, n_reps, L],
    nodes [nSets, n_reps, I]) with the root at I-1."""
    P = np.asarray(P, dtype=np.float64)
    n_sets, B, D = P.shape[0], P.shape[1], P.shape[2]
    fp = np.asarray(flat_parents, dtype=np.int64)
    L = int(n_leaves)
    I = len(fp) - L
    assert B == L + I - 1
    g = np.tile(np.arange(first_rep, first_rep + n_reps, dtype=np.uint64), n_sets)      # [nSets * n_reps], set-major
    t = np.repeat(np.arange(first_set, first_set + n_sets, dtype=np.uint64), n_reps)
    s = np.repeat(np.arange(n_sets), n_reps)
    n = len(g)
    rc, rl = prefix(root_freqs)
    state = np.zeros((L + I, n), dtype=np.int64)
    state[L + I - 1] = draw(np.broadcast_to(rc, (n, D)), np.full(n, rl), uniforms(g, L + I - 1, t, seed))
    cdf, last = prefix(P)                                 # [nSets, B, D, D], [nSets, B, D]
    for node in range(L + I - 2, -1, -1):                 # parents come after their children in flat order
        par = state[L + fp[node]]
        state[node] = draw(cdf[s, node, par], last[s, node, par], uniforms(g, node, t, seed))
    shape = (n_sets, n_reps)
    return state[:L].T.reshape(shape + (L,)), state[L:].T.reshape(shape + (I,))
