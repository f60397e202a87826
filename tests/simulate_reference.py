"""numpy restatement of hb2_simulate's stream (include/hyphy_b200.h): Philox4x32-10, the 53-bit uniform, the draw rule and
the walk from the root.  Fed the engine's own transition matrices it must reproduce the engine's output bit for bit.
No test functions live here."""
import numpy as np

_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)
_MASK = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """ctr [..., 4] and key [..., 2] as unsigned 32-bit words (broadcast against each other); returns [..., 4] uint32."""
    c = [np.asarray(ctr, dtype=np.uint64)[..., i] & _MASK for i in range(4)]
    k = [np.asarray(key, dtype=np.uint64)[..., i] & _MASK for i in range(2)]
    for r in range(10):
        if r > 0:
            k = [(k[0] + _W0) & _MASK, (k[1] + _W1) & _MASK]
        p0, p1 = _M0 * c[0], _M1 * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k[0], p1 & _MASK, (p0 >> np.uint64(32)) ^ c[3] ^ k[1], p0 & _MASK]
    return np.stack(np.broadcast_arrays(*c), axis=-1).astype(np.uint32)


def uniforms(g, slot, seed):
    """u of draw `slot` for global sites g (array): (x0 * 2^21 + (x1 >> 11)) * 2^-53."""
    g = np.asarray(g, dtype=np.uint64)
    seed = np.uint64(seed)
    ctr = np.stack([g & _MASK, g >> np.uint64(32), np.full_like(g, slot), np.zeros_like(g)], axis=-1)
    key = np.array([seed & _MASK, seed >> np.uint64(32)], dtype=np.uint64)
    x = philox4x32_10(ctr, key).astype(np.uint64)
    return ((x[..., 0] << np.uint64(21)) + (x[..., 1] >> np.uint64(11))).astype(np.float64) * 2.0 ** -53


def prefix(v):
    """Sequential fp64 prefix sums over the last axis with entries that are not > 0 counted as 0, and the index of the
    last positive entry (-1 when there is none)."""
    v = np.asarray(v, dtype=np.float64)
    pos = v > 0                                           # False for NaN
    c = np.cumsum(np.where(pos, v, 0.0), axis=-1)         # cumsum adds in order
    m = v.shape[-1]
    last = np.where(pos.any(axis=-1), m - 1 - np.argmax(pos[..., ::-1], axis=-1), -1)
    return c, last


def draw(c, last, u):
    """The draw rule on prefix sums c [n, m] (one row per u) with fall-back indices last [n]."""
    c = np.atleast_2d(c)
    t = u * c[:, -1]
    j = (c <= t[:, None]).sum(axis=1)                     # smallest j with t < c_j (c is non-decreasing)
    return np.where(j < c.shape[1], j, last)


def simulate(P, weights, root_freqs, flat_parents, n_leaves, n_sites, seed, first_site=0):
    """P [C, B, D, D] (row = parent state), weights [C] (None: one class).  Returns (leaf [L, n], nodes [I, n], classes [n])."""
    P = np.asarray(P, dtype=np.float64)
    C, B, D = P.shape[0], P.shape[1], P.shape[2]
    fp = np.asarray(flat_parents, dtype=np.int64)
    L = int(n_leaves)
    I = len(fp) - L
    assert B == L + I - 1
    g = np.arange(first_site, first_site + n_sites, dtype=np.uint64)
    if weights is None:
        assert C == 1
        cls = np.zeros(n_sites, dtype=np.int64)
    else:
        cc, cl = prefix(weights)
        cls = draw(np.broadcast_to(cc, (n_sites, C)), np.full(n_sites, cl), uniforms(g, L + I, seed)) if C > 1 else np.zeros(n_sites, np.int64)
    rc, rl = prefix(root_freqs)
    state = np.zeros((L + I, n_sites), dtype=np.int64)
    state[L + I - 1] = draw(np.broadcast_to(rc, (n_sites, D)), np.full(n_sites, rl), uniforms(g, L + I - 1, seed))
    cdf, last = prefix(P)                                 # [C, B, D, D], [C, B, D]
    for node in range(L + I - 2, -1, -1):                 # parents come after their children in flat order
        par = state[L + fp[node]]
        state[node] = draw(cdf[cls, node, par], last[cls, node, par], uniforms(g, node, seed))
    return state[:L], state[L:], cls.astype(np.int32)
