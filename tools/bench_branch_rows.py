"""MEME's branch-level empirical Bayes rows (hb2_batch_branch_component_likelihoods) on the north-star alignment (200 taxa x
2000 codons, MG94xREV), one set per pattern, in bench_batch_sites.py's MEME shapes:
  meme_all   K = 2 components on every branch
  meme_third K = 2 on a seeded third of the branches, one component elsewhere, tested / background as the group hint
For each shape, with a warm-up call of every size first and medians of --reps blocking calls (host clock):
  * sets/s of the new call and of hb2_batch_site_mixture_likelihoods on the same sets;
  * rows/s of the new call against MEME's brute force -- the mixture entry point fed one set per (set, row) with one-hot
    weights on the row's branch -- on the first --brute-sets sets;
  * in a separate pass under torch.profiler: device time per kernel group (expm pipeline, prune_batch_kernel,
    branch_rows_kernel), and the algorithmic bytes of branch_rows_kernel's matrix reads over its time against 3.35 TB/s.
The card's name and power limit are read in the same run.  One JSON line on stdout; `sha256` fingerprints the rows of
the first call, `max_brute_rel` is the largest relative difference from the brute force."""
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

SHAPES = ("meme_all", "meme_third")
HBM_BYTES_PER_S = 3.35e12            # H100 SXM data sheet


def median_time(call, reps):
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        call()                                                          # returns after the stream is synchronised
        times.append(time.perf_counter() - t0)
    return float(np.median(times)), [min(times), max(times)]


def one_hot_sets(V, W, bk, n):
    """The first n sets as MEME's brute force evaluates them: one set per (set, row), the row's branch one-hot."""
    R = W.shape[1]
    off = np.concatenate([[0], np.cumsum(bk)])
    Wh = np.repeat(W[:n], R, axis=0).reshape(n, R, R)
    for b in range(len(bk)):
        for r in range(off[b], off[b + 1]):
            Wh[:, r, off[b]:off[b + 1]] = 0.0
            Wh[:, r, r] = 1.0
    return np.repeat(V[:n], R, axis=0), Wh.reshape(n * R, R)


def matrix_bytes(w, bk, pats):
    """Bytes of the P area branch_rows_kernel reads, summed over the sets: per component row of an internal child, the D
    rows of 64 doubles of the transposed table for the message and again for the row, and D x D entries for the outside
    vector; per component row of a leaf child, one row of 64 doubles each for message and row (an ambiguous leaf, one
    per allowed state)."""
    D, L = w.D, w.tree.n_leaves
    total = 0
    for p in pats:
        for b in range(w.tree.n_branches):
            if b >= L:
                per = 2 * D * 64 + D * D
            else:
                code = w.leaf_states[b, p]
                per = 2 * 64 * (1 if code >= 0 else int((w.ambig[-code - 1] != 0).sum()))
            total += int(bk[b]) * per * 8
    return total


def profile(lf, w, call, out_dir):
    """Device time per kernel group of one call, from torch.profiler (a pass of its own)."""
    import torch
    from torch.profiler import ProfilerActivity, profile as tprofile
    torch.cuda.init()
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    groups = {"expm": 0.0, "prune_batch_kernel": 0.0, "branch_rows_kernel": 0.0, "other": 0.0}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
        name = e.key
        key = ("branch_rows_kernel" if "branch_rows_kernel" in name else "prune_batch_kernel" if "prune_batch_kernel" in name
               else "expm" if "expm" in name else "other")
        groups[key] += us / 1e6
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "bench_branch_rows_kernels.txt"), "a") as f:
            f.write(prof.key_averages().table(sort_by="device_time_total", row_limit=30) + "\n")
    return groups


def run(lf, w, shape, reps, n_brute, out_dir):
    V, W, bk, bg = make_sets(w, shape)
    if bk is None:
        bk = np.full(w.tree.n_branches, 1, dtype=np.int64)
    pats = np.arange(w.S)
    R = W.shape[1]
    new = lambda: lf.part.batch_branch_component_likelihoods(pats, V, W, w.pi, branch_k=bk, branch_group=bg)    # noqa: E731
    mix = lambda: lf.part.batch_site_mixture_likelihoods(pats, V, W, w.pi, branch_k=bk, branch_group=bg)        # noqa: E731
    Vb, Wb = one_hot_sets(V, W, bk, n_brute)
    pb = np.repeat(pats[:n_brute], R)
    brute = lambda: lf.part.batch_site_mixture_likelihoods(pb, Vb, Wb, w.pi, branch_k=bk, branch_group=bg)      # noqa: E731
    small = lambda: lf.part.batch_branch_component_likelihoods(pats[:n_brute], V[:n_brute], W[:n_brute], w.pi,  # noqa: E731
                                                                branch_k=bk, branch_group=bg)
    site, rows = new()                                                  # warm-up of every size
    mixed = mix()
    ref = brute().reshape(n_brute, R)
    small()
    t_new, s_new = median_time(new, reps)
    t_mix, s_mix = median_time(mix, reps)
    t_brute, s_brute = median_time(brute, max(1, reps // 2))
    t_small, s_small = median_time(small, reps)
    groups = profile(lf, w, new, out_dir)
    rb = matrix_bytes(w, bk, pats)
    kt = groups["branch_rows_kernel"]
    return {"shape": shape, "sets": int(w.S), "rows_per_set": int(R),
            "new_s": t_new, "new_spread_s": s_new, "new_sets_per_s": w.S / t_new, "new_rows_per_s": w.S * R / t_new,
            "mixture_s": t_mix, "mixture_spread_s": s_mix, "mixture_sets_per_s": w.S / t_mix,
            "brute_sets": n_brute, "brute_s": t_brute, "brute_spread_s": s_brute, "brute_rows_per_s": n_brute * R / t_brute,
            "new_subset_s": t_small, "new_subset_spread_s": s_small, "new_subset_rows_per_s": n_brute * R / t_small,
            "kernel_s": groups, "branch_rows_matrix_bytes": rb,
            "branch_rows_bytes_per_s": rb / kt if kt > 0 else None,
            "branch_rows_share_of_hbm": rb / kt / HBM_BYTES_PER_S if kt > 0 else None,
            "site_equals_mixture": bool(np.array_equal(site, mixed)),
            "max_brute_rel": float(np.max(np.abs(rows[:n_brute] - ref) / np.abs(ref))),
            "finite": int(np.isfinite(rows).sum()), "sha256": hashlib.sha256(rows.tobytes()).hexdigest()[:16]}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--brute-sets", type=int, default=6, help="sets of the brute-force comparison")
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
