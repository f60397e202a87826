"""Leaf state imputation (hb2_batch_leaf_support) on the north-star alignment (200 taxa x 2000 codons, MG94xREV), one set
per pattern, in bench_batch_sites.py's shapes:
  fel        one matrix per branch (plain layout), tested / background branches as the group hint
  meme_all   K = 2 components on every branch (mixture layout)
  meme_third K = 2 on a seeded third of the branches, one component elsewhere, tested / background as the group hint
For each shape, with a warm-up call of every size first and medians of --reps blocking calls (host clock):
  * sets/s of the new call and of the likelihood entry point on the same sets (hb2_batch_site_likelihoods or
    hb2_batch_site_mixture_likelihoods);
  * the reference's procedure on the device -- hb2_batch_column_likelihoods fed one column per (leaf, state), L x D
    columns per set -- on the first --brute-sets sets, against the new call on the same sets;
  * in a separate pass under torch.profiler: device time per kernel group (expm pipeline, prune_batch_kernel,
    leaf_support_kernel, the support copy);
  * the bytes of the support copy.
The card's name and power limit are read in the same run.  One JSON line on stdout; `sha256` fingerprints the support of
the first call, `max_brute_rel` is the largest relative difference from the brute force on entries >= 1e-6."""
import argparse
import hashlib
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np  # noqa: E402

from bench_batch_sites import card, make_sets  # noqa: E402
from hyphy_b200 import synth, LikelihoodFunction, engine  # noqa: E402

SHAPES = ("fel", "meme_all", "meme_third")


def median_time(call, reps):
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        call()                                                          # returns after the stream is synchronised
        times.append(time.perf_counter() - t0)
    return float(np.median(times)), [min(times), max(times)]


def forced_columns(w, pats):
    """[len(pats) * L * D, L]: every pattern's column with leaf l forced to state k, row (set, l, k)."""
    L, D = w.tree.n_leaves, w.D
    out = []
    for p in pats:
        c = np.repeat(w.leaf_states[:, p][None, :], L * D, axis=0)
        for l in range(L):
            c[l * D:(l + 1) * D, l] = np.arange(D)
        out.append(c)
    return np.ascontiguousarray(np.concatenate(out))


def profile(call, out_dir):
    """Device time per kernel group of one call, from torch.profiler (a pass of its own)."""
    import torch
    from torch.profiler import ProfilerActivity, profile as tprofile
    torch.cuda.init()
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    groups = {"expm": 0.0, "prune_batch_kernel": 0.0, "leaf_support_kernel": 0.0, "memcpy_dtoh": 0.0, "other": 0.0}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
        name = e.key
        key = ("leaf_support_kernel" if "leaf_support_kernel" in name else "prune_batch_kernel" if "prune_batch_kernel" in name
               else "expm" if "expm" in name else "memcpy_dtoh" if "DtoH" in name or "Device -> Pageable" in name else "other")
        groups[key] += us / 1e6
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "bench_leaf_support_kernels.txt"), "a") as f:
            f.write(prof.key_averages().table(sort_by="device_time_total", row_limit=30) + "\n")
    return groups


def run(lf, w, shape, reps, n_brute, out_dir):
    V, W, bk, bg = make_sets(w, shape)
    L, D = w.tree.n_leaves, w.D
    pats = np.arange(w.S)
    part = lf.part
    new = lambda: part.batch_leaf_support(pats, V, w.pi, weights=W, branch_k=bk, branch_group=bg, want_site=True)  # noqa: E731
    if W is None:
        site_call = lambda: part.batch_site_likelihoods(pats, V, w.pi, branch_group=bg)       # noqa: E731
    else:
        site_call = lambda: part.batch_site_mixture_likelihoods(pats, V, W, w.pi, branch_k=bk, branch_group=bg)  # noqa: E731
    cols = forced_columns(w, pats[:n_brute])
    per = L * D
    Vb = np.repeat(V[:n_brute], per, axis=0)
    Wb = None if W is None else np.repeat(W[:n_brute], per, axis=0)
    brute = lambda: part.batch_column_likelihoods(cols, Vb, w.pi, weights=Wb, branch_k=bk, branch_group=bg)  # noqa: E731
    small = lambda: part.batch_leaf_support(pats[:n_brute], V[:n_brute], w.pi, weights=None if W is None else W[:n_brute],  # noqa: E731
                                            branch_k=bk, branch_group=bg)
    sup, site = new()                                                   # warm-up of every size
    lnl = site_call()
    b = brute().reshape(n_brute, L, D)
    small()
    t_new, s_new = median_time(new, reps)
    t_site, s_site = median_time(site_call, reps)
    t_brute, s_brute = median_time(brute, max(1, reps // 2))
    t_small, s_small = median_time(small, reps)
    groups = profile(new, out_dir)
    x = np.exp(b - b.max(axis=2, keepdims=True))
    ref = x / x.sum(axis=2, keepdims=True)
    big = ref >= 1e-6
    return {"shape": shape, "sets": int(w.S), "leaves": L, "states": D,
            "new_s": t_new, "new_spread_s": s_new, "new_sets_per_s": w.S / t_new,
            "site_call_s": t_site, "site_call_spread_s": s_site, "site_call_sets_per_s": w.S / t_site,
            "new_over_site_call": t_new / t_site,
            "brute_sets": n_brute, "brute_columns": int(len(cols)), "brute_s": t_brute, "brute_spread_s": s_brute,
            "new_subset_s": t_small, "new_subset_spread_s": s_small, "brute_over_new_subset": t_brute / t_small,
            "kernel_s": groups, "support_copy_bytes": int(sup.nbytes),
            "site_equals_site_call": bool(np.array_equal(site, lnl)),
            "max_brute_rel": float(np.max(np.abs(sup[:n_brute][big] - ref[big]) / ref[big])),
            "max_row_sum_err": float(np.abs(sup.sum(axis=2) - 1).max()),
            "finite": int(np.isfinite(sup).sum()), "sha256": hashlib.sha256(sup.tobytes()).hexdigest()[:16]}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--brute-sets", type=int, default=1, help="sets of the brute-force comparison (L x D columns each)")
    ap.add_argument("--shapes", default=",".join(SHAPES), help="comma-separated subset of " + ", ".join(SHAPES))
    ap.add_argument("--profile-dir", default=None, help="where to write the profiler's kernel table (optional)")
    args = ap.parse_args()
    if engine.device_count() < 1:
        sys.exit("no CUDA device: this benchmark measures the GPU and has nothing to fall back to")
    info = card()
    w = synth.codon_workload(200, 2000, 1)
    lf = LikelihoodFunction(w, flags=engine.FLAG_FORCE_FP64)
    lf.set_template()
    out = dict(info, workload=f"MG94xREV {w.tree.n_leaves}x2000, {w.S} patterns, {w.tree.n_branches} branches", results=[])
    for shape in args.shapes.split(","):
        out["results"].append(run(lf, w, shape, args.reps, args.brute_sets, args.profile_dir))
    lf.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
