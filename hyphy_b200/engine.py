"""Host-side mirror of the reference's evaluator interface over the C ABI (ctypes; no torch types involved).

`Partition` is a 1:1 wrapper of include/hyphy_b200.h.  `LikelihoodFunction` mirrors the slice of
`_LikelihoodFunction` the hot path touches (likefunc.cpp): SetupLFCaches -> constructor, ExponentiateMatrices ->
set_matrices, ComputeBlock(index, siteRes, currentRateClass) -> compute_block, Compute -> compute,
DeleteCaches -> close.  There is NO CPU fallback: if the CUDA library or a GPU is missing every entry raises.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("HB2_LIB") or os.path.join(PKG, "libhyphy_b200.so")   # HB2_LIB: A/B another build of the engine

MATRIX_RATE = 0
MATRIX_TRANS = 1
FLAG_DEFAULT = 0
FLAG_FORCE_FP64 = 1

_dp = C.POINTER(C.c_double)
_ip = C.POINTER(C.c_int64)
_i32p = C.POINTER(C.c_int32)

# every symbol include/hyphy_b200.h declares: (name, restype, argtypes)
ABI = [
    ("hb2_abi_version", C.c_int, []),
    ("hb2_last_error", C.c_char_p, []),
    ("hb2_device_count", C.c_int, []),
    ("hb2_create", C.c_int, [C.POINTER(C.c_void_p), C.c_int64, C.c_int64, C.c_int64, C.c_int64, C.c_int64, _ip, _ip, _dp,
                             C.c_int64, _ip, C.c_int, C.c_int]),
    ("hb2_set_matrices", C.c_int, [C.c_void_p, C.c_int64, C.c_int64, _ip, C.POINTER(_dp), C.c_int]),
    ("hb2_set_matrices_packed", C.c_int, [C.c_void_p, C.c_int64, C.c_int64, _ip, _dp, C.c_int]),
    ("hb2_set_rate_template", C.c_int, [C.c_void_p, C.c_int64, _ip, _ip, C.c_int64, _dp]),
    ("hb2_set_matrices_compiled", C.c_int, [C.c_void_p, C.c_int64, C.c_int64, _ip, _dp]),
    ("hb2_set_rate_template_id", C.c_int, [C.c_void_p, C.c_int64, C.c_int64, _ip, _ip, C.c_int64, _dp]),
    ("hb2_set_matrices_compiled_id", C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int64, _ip, _dp]),
    ("hb2_set_template_frequencies", C.c_int, [C.c_void_p, C.c_int64, _dp]),
    ("hb2_set_mixture_matrices", C.c_int, [C.c_void_p, C.c_int64, C.c_int64, _ip, C.c_int64, _dp, _dp]),
    ("hb2_evaluate", C.c_int, [C.c_void_p, C.c_int64, C.c_int64, _ip, _dp, _dp, _dp, _ip]),
    ("hb2_evaluate_forced", C.c_int, [C.c_void_p, C.c_int64, C.c_int64, _ip, _dp, C.c_int64, _ip, _dp, _dp, _ip]),
    ("hb2_evaluate_classes", C.c_int, [C.c_void_p, _dp, C.c_int64, _ip, _dp, _dp, _dp, _ip]),
    ("hb2_batch_site_likelihoods", C.c_int, [C.c_void_p, C.c_int64, C.c_int64, _ip, _dp, _ip, _dp, _dp]),
    ("hb2_batch_site_mixture_likelihoods", C.c_int, [C.c_void_p, C.c_int64, C.c_int64, _ip, C.c_int64, _ip, _dp, _dp, _ip, _dp, _dp]),
    ("hb2_batch_branch_component_likelihoods", C.c_int, [C.c_void_p, C.c_int64, C.c_int64, _ip, C.c_int64, _ip, _dp, _dp, _ip,
                                                         _dp, _dp, _dp]),
    ("hb2_batch_leaf_support", C.c_int, [C.c_void_p, C.c_int64, C.c_int64, _ip, C.c_int64, _ip, _dp, _dp, _ip, _dp, _dp, _dp]),
    ("hb2_batch_joint_ancestors", C.c_int, [C.c_void_p, C.c_int64, C.c_int64, _ip, C.c_int64, _ip, _dp, _dp, _ip, _dp, _dp, _dp,
                                            _ip]),
    ("hb2_batch_column_likelihoods", C.c_int, [C.c_void_p, C.c_int64, C.c_int64, _ip, C.c_int64, _ip, _dp, _dp, _ip, _dp, _dp]),
    ("hb2_batch_site_rates", C.c_int, [C.c_void_p, C.c_int64, C.c_int64, _ip, _dp, _dp, _dp]),
    ("hb2_read_conditionals", C.c_int, [C.c_void_p, C.c_int64, C.c_int64, _dp, _i32p]),
    ("hb2_read_transition", C.c_int, [C.c_void_p, C.c_int64, C.c_int64, _dp]),
    ("hb2_simulate", C.c_int, [C.c_void_p, _dp, _dp, C.c_int64, C.c_uint64, C.c_int64, _ip, _ip, _i32p]),
    ("hb2_batch_site_simulate", C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int64, _ip, _dp, _dp, _ip, _dp, C.c_int64,
                                          C.c_uint64, C.c_int64, C.c_int64, _ip, _ip]),
    ("hb2_comm_unique_id", C.c_int, [C.c_void_p]),
    ("hb2_branch_cache_build", C.c_int, [C.c_void_p, C.c_int64, _dp]),
    ("hb2_branch_cache_evaluate", C.c_int, [C.c_void_p, C.c_int64, _dp, C.POINTER(C.c_double), _dp, _ip]),
    ("hb2_plan_walk", C.c_int, [C.c_int64, C.c_int64, _ip, C.c_int64, _ip, C.c_int, C.c_int, _i32p, _i32p, C.c_int64, _ip]),
    ("hb2_comm_init", C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    ("hb2_comm_class_groups", C.c_int, [C.c_void_p, C.c_int]),
    ("hb2_comm_gather_sites", C.c_int, [C.c_void_p, _dp, _ip, _dp, _ip, C.c_int64, C.POINTER(C.c_int64)]),
    ("hb2_destroy", None, [C.c_void_p]),
    ("hb2_launch_count", C.c_int64, [C.c_void_p]),
    ("hb2_precision_mode", C.c_int, [C.c_void_p]),
    ("hb2_pruning_kernel", C.c_char_p, [C.c_void_p]),
    ("hb2_stage_launches", C.c_int, [C.c_void_p, _ip]),
    ("hb2_time_resident", C.c_int, [C.c_void_p, _dp, _dp, C.c_int, _dp, _dp, _dp]),
]


class EngineError(RuntimeError):
    pass


_lib = None


def load_library():
    """Loads libhyphy_b200.so.  Raises (never falls back) when the CUDA extension has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise EngineError(f"{LIB_PATH} is missing: build it with `python -m hyphy_b200.build` "
                              "(the engine has no CPU fallback)")
        lib = C.CDLL(LIB_PATH)
        for name, res, args in ABI:
            fn = getattr(lib, name)          # AttributeError if the library does not export the symbol
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


STEP_WAIT, STEP_CHAIN, STEP_MUL, STEP_ID_MASK = 1 << 30, 1 << 29, 1 << 28, (1 << 27) - 1
STEP_FIRST, STEP_LAST = 1 << 28, 1 << 29


def plan_walk(flat_parents, n_leaves, update_nodes=None, lanes=4, split_nodes=True, canonical_multi=False):
    """The walk kernel's plan for a tree and a dirty set (host code only: works without a GPU).
    Returns (lane_start[lanes+1], steps[n, 2])."""
    fp, pfp = _i(flat_parents)
    L = int(n_leaves)
    I = len(fp) - L
    ls = np.zeros(lanes + 1, dtype=np.int32)
    st = np.zeros(2 * (L + 2 * I), dtype=np.int32)
    n = C.c_int64()
    if update_nodes is None:
        nu, pu = -1, None
    else:
        u, pu = _i(update_nodes)
        nu = len(u)
    _check(load_library().hb2_plan_walk(L, I, pfp, nu, pu, int(lanes), int(bool(split_nodes)) | (2 if canonical_multi else 0), ls.ctypes.data_as(_i32p),
                                        st.ctypes.data_as(_i32p), len(st) // 2, C.byref(n)))
    return ls, st[:2 * n.value].reshape(-1, 2).copy()


def device_count() -> int:
    return int(load_library().hb2_device_count())


def _check(rc: int):
    if rc != 0:
        raise EngineError(load_library().hb2_last_error().decode("utf-8", "replace"))


def _d(a):
    a = np.ascontiguousarray(a, dtype=np.float64)
    return a, a.ctypes.data_as(_dp)


def _i(a):
    a = np.ascontiguousarray(a, dtype=np.int64)
    return a, a.ctypes.data_as(_ip)


class Partition:
    """One (likelihood function, partition) pair resident on one GPU (opaque hb2_partition handle)."""

    def __init__(self, S, D, L, I, C_, flat_parents, leaf_states, ambig, pattern_freq, device=0, flags=FLAG_DEFAULT):
        self._lib = load_library()
        self.S, self.D, self.L, self.I, self.C = int(S), int(D), int(L), int(I), int(C_)
        self.B = self.L + self.I - 1
        fp, pfp = _i(flat_parents)
        ls, pls = _i(leaf_states)
        fr, pfr = _i(pattern_freq)
        ambig = np.zeros((0, self.D)) if ambig is None else np.asarray(ambig, dtype=np.float64)
        am, pam = _d(ambig if len(ambig) else np.zeros((1, self.D)))
        assert fp.shape == (self.L + self.I,) and ls.shape == (self.L, self.S) and fr.shape == (self.S,)
        h = C.c_void_p()
        _check(self._lib.hb2_create(C.byref(h), self.S, self.D, self.L, self.I, self.C, pfp, pls, pam, len(ambig), pfr,
                                    int(device), int(flags)))
        self._h = h

    # -- ExponentiateMatrices / SetCompExp ---------------------------------------------------------
    def set_matrices(self, cat, node_ids, M, kind=MATRIX_RATE):
        """M: array [n, D, D] (packed).  kind: MATRIX_RATE (Q*t, exponentiated on device) or MATRIX_TRANS (P)."""
        ids, pids = _i(node_ids)
        Mm, pM = _d(M)
        assert Mm.shape == (len(ids), self.D, self.D)
        _check(self._lib.hb2_set_matrices_packed(self._h, int(cat), len(ids), pids, pM, int(kind)))

    def set_matrices_ptrs(self, cat, node_ids, mats, kind=MATRIX_RATE):
        """Pointer-array variant (one D*D matrix per node, as the reference holds them)."""
        ids, pids = _i(node_ids)
        keep = [np.ascontiguousarray(m, dtype=np.float64) for m in mats]
        arr = (_dp * len(keep))(*[m.ctypes.data_as(_dp) for m in keep])
        _check(self._lib.hb2_set_matrices(self._h, int(cat), len(ids), pids, arr, int(kind)))

    def set_rate_template(self, entry_index, entry_formula, n_formulas, col_freq=None):
        ei, pei = _i(entry_index)
        ef, pef = _i(entry_formula)
        assert ei.shape == ef.shape
        pcf = None
        if col_freq is not None:
            cf, pcf = _d(col_freq)
            assert cf.shape == (self.D,)
        self.n_formulas = int(n_formulas)
        _check(self._lib.hb2_set_rate_template(self._h, len(ei), pei, pef, int(n_formulas), pcf))

    def set_matrices_compiled(self, cat, node_ids, values, template=0):
        ids, pids = _i(node_ids)
        v, pv = _d(values)
        assert v.shape[0] == len(ids)
        _check(self._lib.hb2_set_matrices_compiled_id(self._h, int(template), int(cat), len(ids), pids, pv))

    def set_rate_template_id(self, template, entry_index, entry_formula, n_formulas, col_freq=None):
        ei, pei = _i(entry_index)
        ef, pef = _i(entry_formula)
        pcf = None
        if col_freq is not None:
            cf, pcf = _d(col_freq)
        _check(self._lib.hb2_set_rate_template_id(self._h, int(template), len(ei), pei, pef, int(n_formulas), pcf))

    def set_template_frequencies(self, template, col_freq):
        cf, pcf = _d(col_freq)
        _check(self._lib.hb2_set_template_frequencies(self._h, int(template), pcf))

    def set_mixture_matrices(self, cat, node_ids, M, w):
        ids, pids = _i(node_ids)
        Mm, pM = _d(M)
        ww, pw = _d(w)
        assert Mm.ndim == 4 and Mm.shape[0] == len(ids) and ww.shape == Mm.shape[:2]
        _check(self._lib.hb2_set_mixture_matrices(self._h, int(cat), len(ids), pids, Mm.shape[1], pM, pw))

    # -- ComputeBlock ------------------------------------------------------------------------------
    def _eval(self, fn, first, update_nodes, root_freqs, want_sites):
        pi, ppi = _d(root_freqs)
        assert pi.shape == (self.D,)
        if update_nodes is None:
            n, pu = -1, None
        else:
            u, pu = _i(update_nodes)
            n = len(u)
        lnl = C.c_double()
        sl = np.empty(self.S) if want_sites else None
        ss = np.empty(self.S, dtype=np.int64) if want_sites else None
        _check(fn(self._h, first, n, pu, ppi, C.byref(lnl), sl.ctypes.data_as(_dp) if want_sites else None,
                  ss.ctypes.data_as(_ip) if want_sites else None))
        return (lnl.value, sl, ss) if want_sites else lnl.value

    def evaluate(self, cat, root_freqs, update_nodes=None, want_sites=False):
        return self._eval(self._lib.hb2_evaluate, C.c_int64(int(cat)), update_nodes, root_freqs, want_sites)

    def evaluate_forced(self, cat, root_freqs, forced_node, forced_states, update_nodes=None, want_sites=True):
        """ComputeBlock(index, siteRes, cat, branchIndex, branchValues): one node pinned to a state per pattern."""
        pi, ppi = _d(root_freqs)
        fs, pfs = _i(forced_states)
        assert fs.shape == (self.S,)
        if update_nodes is None:
            n, pu = -1, None
        else:
            u, pu = _i(update_nodes)
            n = len(u)
        lnl = C.c_double()
        sl = np.empty(self.S) if want_sites else None
        ss = np.empty(self.S, dtype=np.int64) if want_sites else None
        _check(self._lib.hb2_evaluate_forced(self._h, int(cat), n, pu, ppi, int(forced_node), pfs, C.byref(lnl),
                                             sl.ctypes.data_as(_dp) if want_sites else None, ss.ctypes.data_as(_ip) if want_sites else None))
        return (lnl.value, sl, ss) if want_sites else lnl.value

    def evaluate_classes(self, weights, root_freqs, update_nodes=None, want_sites=False):
        w, pw = _d(weights)
        assert w.shape == (self.C,)
        return self._eval(self._lib.hb2_evaluate_classes, pw, update_nodes, root_freqs, want_sites)

    # -- single-branch shortcut ----------------------------------------------------------------------
    def branch_cache_build(self, node, root_freqs):
        pi, ppi = _d(root_freqs)
        assert pi.shape == (self.D,)
        _check(self._lib.hb2_branch_cache_build(self._h, int(node), ppi))

    def branch_cache_evaluate(self, weights=None, cat=0, want_sites=False):
        """lnL with only the cached branch's matrix changed; weights=None -> single class `cat`."""
        pw = None
        if weights is not None:
            w, pw = _d(weights)
            assert w.shape == (self.C,)
        lnl = C.c_double()
        sl = np.empty(self.S) if want_sites else None
        ss = np.empty(self.S, dtype=np.int64) if want_sites else None
        _check(self._lib.hb2_branch_cache_evaluate(self._h, int(cat), pw, C.byref(lnl), sl.ctypes.data_as(_dp) if want_sites else None,
                                                   ss.ctypes.data_as(_ip) if want_sites else None))
        return (lnl.value, sl, ss) if want_sites else lnl.value

    # -- batched one-pattern likelihoods (FEL / MEME site phases) -------------------------------------
    def batch_site_likelihoods(self, pattern_of, formula_values, root_freqs, branch_group=None, template=0):
        """formula_values: [nSets, B, nF]; returns the nSets log-likelihoods."""
        po, ppo = _i(pattern_of)
        _, _, pv, _, pbg, keep = self._batch_rows(len(po), formula_values, None, None, branch_group)
        pi, ppi = _d(root_freqs)
        out = np.empty(len(po))
        _check(self._lib.hb2_batch_site_likelihoods(self._h, int(template), len(po), ppo, pv, pbg, ppi, out.ctypes.data_as(_dp)))
        return out

    def batch_site_mixture_likelihoods(self, pattern_of, formula_values, weights, root_freqs, branch_k=None, branch_group=None,
                                       template=0):
        """MEME's site model: branch b mixes branch_k[b] components (None: weights.shape[1] / B on every branch).
        formula_values: [nSets, R, nF], weights: [nSets, R], R = sum of branch_k; returns the nSets log-likelihoods."""
        po, ppo = _i(pattern_of)
        assert weights is not None
        K, pbk, pv, pw, pbg, keep = self._batch_rows(len(po), formula_values, weights, branch_k, branch_group)
        pi, ppi = _d(root_freqs)
        out = np.empty(len(po))
        _check(self._lib.hb2_batch_site_mixture_likelihoods(self._h, int(template), len(po), ppo, K, pbk, pv, pw, pbg, ppi,
                                                            out.ctypes.data_as(_dp)))
        return out

    def batch_branch_component_likelihoods(self, pattern_of, formula_values, weights, root_freqs, branch_k=None,
                                           branch_group=None, template=0):
        """MEME's branch-level empirical Bayes (hb2_batch_branch_component_likelihoods): arguments as
        batch_site_mixture_likelihoods.  Returns (site_lnl [nSets], row_lnl [nSets, R]): row r of a set is its log-likelihood
        with that row's branch pinned to that row's component alone."""
        po, ppo = _i(pattern_of)
        assert weights is not None
        K, pbk, pv, pw, pbg, keep = self._batch_rows(len(po), formula_values, weights, branch_k, branch_group)
        pi, ppi = _d(root_freqs)
        site = np.empty(len(po))
        rows = np.empty((len(po), keep[1].shape[1]))
        _check(self._lib.hb2_batch_branch_component_likelihoods(self._h, int(template), len(po), ppo, K, pbk, pv, pw, pbg, ppi,
                                                                site.ctypes.data_as(_dp), rows.ctypes.data_as(_dp)))
        return site, rows

    def batch_leaf_support(self, pattern_of, formula_values, root_freqs, weights=None, branch_k=None, branch_group=None,
                           template=0, want_site=False):
        """Leaf state imputation (hb2_batch_leaf_support): sets as batch_column_likelihoods on partition patterns.  Returns
        support [nSets, L, D], row l of a set being the distribution of leaf l's state given every other leaf; with
        want_site also the nSets site log-likelihoods, as (support, site_lnl)."""
        po, ppo = _i(pattern_of)
        K, pbk, pv, pw, pbg, keep = self._batch_rows(len(po), formula_values, weights, branch_k, branch_group)
        pi, ppi = _d(root_freqs)
        site = np.empty(len(po)) if want_site else None
        sup = np.empty((len(po), self.L, self.D))
        _check(self._lib.hb2_batch_leaf_support(self._h, int(template), len(po), ppo, K, pbk, pv, pw, pbg, ppi,
                                                site.ctypes.data_as(_dp) if want_site else None, sup.ctypes.data_as(_dp)))
        return (sup, site) if want_site else sup

    def batch_joint_ancestors(self, pattern_of, formula_values, root_freqs, weights=None, branch_k=None, branch_group=None,
                              template=0, want_site=False):
        """Joint maximum-likelihood ancestral states (hb2_batch_joint_ancestors): sets as batch_leaf_support.  Returns
        (node_states [nSets, I], joint_lnl [nSets]), node_states[s][i] being internal node i's state or -1 (unresolved);
        with want_site also the nSets site log-likelihoods, as (node_states, joint_lnl, site_lnl)."""
        po, ppo = _i(pattern_of)
        K, pbk, pv, pw, pbg, keep = self._batch_rows(len(po), formula_values, weights, branch_k, branch_group)
        pi, ppi = _d(root_freqs)
        site = np.empty(len(po)) if want_site else None
        jl = np.empty(len(po))
        st = np.empty((len(po), self.I), dtype=np.int64)
        _check(self._lib.hb2_batch_joint_ancestors(self._h, int(template), len(po), ppo, K, pbk, pv, pw, pbg, ppi,
                                                   site.ctypes.data_as(_dp) if want_site else None, jl.ctypes.data_as(_dp),
                                                   st.ctypes.data_as(_ip)))
        return (st, jl, site) if want_site else (st, jl)

    def _batch_rows(self, n_sets, formula_values, weights, branch_k, branch_group):
        """Checked arguments of the batch entry points that take both set layouts: weights None means one row per branch
        (formula_values [nSets, B, nF]); otherwise as batch_site_mixture_likelihoods."""
        v, pv = _d(formula_values)
        assert v.ndim == 3 and v.shape[0] == n_sets
        K, pw, pbk, pbg, keep = 1, None, None, None, [v]
        if weights is None:
            assert branch_k is None and v.shape[1] == self.B
        else:
            w, pw = _d(weights)
            assert w.shape == v.shape[:2]
            keep.append(w)
            if branch_k is None:
                assert w.shape[1] % self.B == 0
                K = w.shape[1] // self.B
            else:
                bk, pbk = _i(branch_k)
                assert bk.shape == (self.B,) and bk.sum() == w.shape[1]
                K = int(bk.max())
                keep.append(bk)
        if branch_group is not None:
            bg, pbg = _i(branch_group)
            assert bg.shape == (self.B,)
            keep.append(bg)
        return K, pbk, pv, pw, pbg, keep

    def batch_column_likelihoods(self, columns, formula_values, root_freqs, weights=None, branch_k=None, branch_group=None,
                                 template=0):
        """Batch likelihoods of caller-given columns [nSets, L] (hb2_create's leaf codes) instead of partition patterns;
        sets as batch_site_likelihoods (weights None) or batch_site_mixture_likelihoods.  Returns the nSets log-likelihoods."""
        col, pcol = _i(columns)
        assert col.ndim == 2 and col.shape[1] == self.L
        K, pbk, pv, pw, pbg, keep = self._batch_rows(len(col), formula_values, weights, branch_k, branch_group)
        pi, ppi = _d(root_freqs)
        out = np.empty(len(col))
        _check(self._lib.hb2_batch_column_likelihoods(self._h, int(template), len(col), pcol, K, pbk, pv, pw, pbg, ppi,
                                                      out.ctypes.data_as(_dp)))
        return out

    def batch_site_simulate(self, formula_values, root_freqs, n_reps, weights=None, branch_k=None, branch_group=None, seed=0,
                            first_set=0, first_rep=0, want_nodes=False, template=0):
        """Replicates first_rep .. first_rep + n_reps - 1 of sets first_set .. of the stream `seed`, each simulated from its
        own set's model (hb2_batch_site_simulate); sets as batch_column_likelihoods.  Returns (leaf states
        [nSets, n_reps, L] int64, internal-node states [nSets, n_reps, I] int64 or None)."""
        v = np.asarray(formula_values)
        n = len(v)
        K, pbk, pv, pw, pbg, keep = self._batch_rows(n, v, weights, branch_k, branch_group)
        pi, ppi = _d(root_freqs)
        assert pi.shape == (self.D,)
        r = max(int(n_reps), 0)
        leaf = np.empty((n, r, self.L), dtype=np.int64)
        nodes = np.empty((n, r, self.I), dtype=np.int64) if want_nodes else None
        _check(self._lib.hb2_batch_site_simulate(self._h, int(template), n, K, pbk, pv, pw, pbg, ppi, int(n_reps),
                                                 int(seed) & 0xFFFFFFFFFFFFFFFF, int(first_set), int(first_rep),
                                                 leaf.ctypes.data_as(_ip), nodes.ctypes.data_as(_ip) if want_nodes else None))
        return leaf, nodes

    def batch_site_rates(self, pattern_of, rates, root_freqs, cat=0):
        """LEISR's site model (hb2_batch_site_rates): set s is pattern pattern_of[s] under class `cat` of the current model
        with every branch's rate matrix multiplied by rates[s].  Returns the nSets log-likelihoods."""
        po, ppo = _i(pattern_of)
        r, pr = _d(rates)
        assert po.ndim == 1 and r.shape == po.shape
        pi, ppi = _d(root_freqs)
        assert pi.shape == (self.D,)
        out = np.empty(len(po))
        _check(self._lib.hb2_batch_site_rates(self._h, int(cat), len(po), ppo, pr, ppi, out.ctypes.data_as(_dp)))
        return out

    # -- read-backs --------------------------------------------------------------------------------
    def read_conditionals(self, cat, inode):
        cond = np.empty((self.S, self.D))
        e = np.empty(self.S, dtype=np.int32)
        _check(self._lib.hb2_read_conditionals(self._h, int(cat), int(inode), cond.ctypes.data_as(_dp), e.ctypes.data_as(_i32p)))
        return cond, e

    def read_transition(self, cat, node):
        P = np.empty((self.D, self.D))
        _check(self._lib.hb2_read_transition(self._h, int(cat), int(node), P.ctypes.data_as(_dp)))
        return P

    # -- SimulateDataSet ---------------------------------------------------------------------------
    def simulate(self, n_sites, root_freqs, weights=None, seed=0, first_site=0, want_nodes=False, want_classes=False):
        """Sites first_site .. first_site + n_sites - 1 of the simulation stream `seed` (hb2_simulate) from the current
        matrices.  Returns (leaf states [L, n] int64, internal-node states [I, n] int64 or None, classes [n] int32 or None)."""
        n = int(n_sites)
        pi, ppi = _d(root_freqs)
        assert pi.shape == (self.D,)
        pw = None
        if weights is not None:
            w, pw = _d(weights)
            assert w.shape == (self.C,)
        leaf = np.empty((self.L, max(n, 0)), dtype=np.int64)
        nodes = np.empty((self.I, max(n, 0)), dtype=np.int64) if want_nodes else None
        classes = np.empty(max(n, 0), dtype=np.int32) if want_classes else None
        _check(self._lib.hb2_simulate(self._h, pw, ppi, n, int(seed) & 0xFFFFFFFFFFFFFFFF, int(first_site), leaf.ctypes.data_as(_ip),
                                      nodes.ctypes.data_as(_ip) if want_nodes else None,
                                      classes.ctypes.data_as(_i32p) if want_classes else None))
        return leaf, nodes, classes

    # -- multi-GPU ---------------------------------------------------------------------------------
    @staticmethod
    def comm_unique_id() -> bytes:
        buf = C.create_string_buffer(128)
        _check(load_library().hb2_comm_unique_id(buf))
        return buf.raw

    def comm_init(self, n_ranks: int, rank: int, unique_id: bytes):
        assert len(unique_id) == 128
        buf = C.create_string_buffer(unique_id, 128)
        _check(self._lib.hb2_comm_init(self._h, int(n_ranks), int(rank), buf))

    def comm_class_groups(self, n_groups: int):
        """Second sharding axis (rate classes); see hb2_comm_class_groups in include/hyphy_b200.h."""
        _check(self._lib.hb2_comm_class_groups(self._h, int(n_groups)))

    def comm_gather_sites(self, site_l, site_scale, capacity: int):
        """All shards' per-pattern outputs on every rank (hb2_comm_gather_sites); returns (siteL, siteScale) of the whole alignment."""
        sl = np.ascontiguousarray(site_l, dtype=np.float64)
        ss = np.ascontiguousarray(site_scale, dtype=np.int64)
        out_l = np.empty(int(capacity))
        out_s = np.empty(int(capacity), dtype=np.int64)
        tot = C.c_int64()
        _check(self._lib.hb2_comm_gather_sites(self._h, sl.ctypes.data_as(_dp), ss.ctypes.data_as(_ip), out_l.ctypes.data_as(_dp),
                                               out_s.ctypes.data_as(_ip), int(capacity), C.byref(tot)))
        return out_l[:tot.value], out_s[:tot.value]

    # -- introspection -----------------------------------------------------------------------------
    @property
    def launch_count(self) -> int:
        return int(self._lib.hb2_launch_count(self._h))

    @property
    def precision_mode(self) -> int:
        return int(self._lib.hb2_precision_mode(self._h))

    @property
    def pruning_kernel(self) -> str:
        return self._lib.hb2_pruning_kernel(self._h).decode()

    @property
    def stage_launches(self):
        out = np.zeros(3, dtype=np.int64)
        _check(self._lib.hb2_stage_launches(self._h, out.ctypes.data_as(_ip)))
        return out

    def time_resident(self, weights, root_freqs, iters=10):
        w, pw = _d(weights)
        pi, ppi = _d(root_freqs)
        ms, lnl = C.c_double(), C.c_double()
        st = np.zeros(3)
        _check(self._lib.hb2_time_resident(self._h, pw, ppi, int(iters), C.byref(ms), st.ctypes.data_as(_dp), C.byref(lnl)))
        return ms.value, st, lnl.value

    def close(self):
        if getattr(self, "_h", None):
            self._lib.hb2_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class LikelihoodFunction:
    """Mirror of the `_LikelihoodFunction` slice on the hot path, for ONE partition of a workload
    (hyphy_b200.synth.Workload or anything with the same fields).

      __init__           SetupLFCaches        likefunc.cpp:4163
      set_all_matrices   ExponentiateMatrices tree.cpp:2932 (every branch, every rate class)
      compute_block      ComputeBlock         likefunc.cpp:10783 (one rate class; optional per-pattern outputs)
      compute            Compute              likefunc.cpp:2421 (category path fused on device)
      simulate           SimulateDataSet      likefunc.cpp:12584 (discrete-category mode)
      close              DeleteCaches         likefunc.cpp:10556
    """

    def __init__(self, w, device=0, flags=FLAG_DEFAULT, pattern_slice: slice | None = None):
        self.w = w
        t = w.tree
        ls, fr = w.leaf_states, w.pattern_freq
        if pattern_slice is not None:                       # multi-GPU pattern shard
            ls, fr = ls[:, pattern_slice], fr[pattern_slice]
        self.part = Partition(ls.shape[1], w.D, t.n_leaves, t.n_internal, w.C, t.flat_parents, ls, w.ambig, fr, device, flags)
        self.all_nodes = np.arange(t.n_branches, dtype=np.int64)

    def set_all_matrices(self, Qt=None, kind=MATRIX_RATE):
        Qt = self.w.Qt() if Qt is None else Qt
        for c in range(self.w.C):
            self.part.set_matrices(c, self.all_nodes, Qt[c], kind)

    def set_template(self):
        """Hand the model's compiled template over once (the static half of _CompiledMatrixData)."""
        ei, ef, nf, cf = self.w.compiled_template()
        self.part.set_rate_template(ei, ef, nf, cf)

    def set_all_compiled(self, values=None):
        """Per-evaluation half: formula values [C, B, nF] for every branch and class."""
        values = self.w.compiled_values() if values is None else values
        for c in range(self.w.C):
            self.part.set_matrices_compiled(c, self.all_nodes, values[c])

    def compute_block(self, cat=0, update_nodes=None, want_sites=False):
        return self.part.evaluate(cat, self.w.pi, update_nodes, want_sites)

    def compute(self, update_nodes=None, want_sites=False, weights=None):
        wts = self.w.class_weights if weights is None else weights
        return self.part.evaluate_classes(wts, self.w.pi, update_nodes, want_sites)

    def simulate(self, n_sites, seed=0, first_site=0, want_nodes=False, want_classes=False):
        """SimulateDataSet from the current matrices with the workload's root frequencies and class weights:
        (leaf states [L, n], internal-node states [I, n] | None, classes [n] | None); see Partition.simulate."""
        return self.part.simulate(n_sites, self.w.pi, self.w.class_weights, seed, first_site, want_nodes, want_classes)

    def close(self):
        self.part.close()
