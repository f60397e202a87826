"""Joint maximum-likelihood ancestral states (hb2_batch_joint_ancestors) on the north-star alignment (200 taxa x 2000
codons, MG94xREV), one set per pattern, in bench_batch_sites.py's shapes:
  fel        one matrix per branch (plain layout), tested / background branches as the group hint
  meme_all   K = 2 components on every branch (mixture layout)
  meme_third K = 2 on a seeded third of the branches, one component elsewhere, tested / background as the group hint
For each shape, with a warm-up call first and medians of --reps blocking calls (host clock):
  * sets/s of the new call (without siteLnL, as a caller that already has the likelihoods makes it) and of the
    likelihood entry point on the same sets (hb2_batch_site_likelihoods or hb2_batch_site_mixture_likelihoods);
  * in a separate pass under torch.profiler: device time per kernel group (expm pipeline, prune_batch_kernel,
    joint_ancestors_kernel, copies), from one call with siteLnL so that both pruning kernels run on the same sets.
The card's name and power limit are read in the same run.  One JSON line on stdout; `sha256_states` and `sha256_lnl`
fingerprint nodeStates and jointLnL of the first call."""
import argparse
import hashlib
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np  # noqa: E402

from bench_batch_sites import card, make_sets  # noqa: E402
from bench_leaf_support import median_time  # noqa: E402
from hyphy_b200 import synth, LikelihoodFunction, engine  # noqa: E402

SHAPES = ("fel", "meme_all", "meme_third")


def profile(call, out_dir):
    """Device time per kernel group of one call, from torch.profiler (a pass of its own)."""
    import torch
    from torch.profiler import ProfilerActivity, profile as tprofile
    torch.cuda.init()
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    groups = {"expm": 0.0, "prune_batch_kernel": 0.0, "joint_ancestors_kernel": 0.0, "memcpy": 0.0, "other": 0.0}
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
        name = e.key
        key = ("joint_ancestors_kernel" if "joint_ancestors_kernel" in name else "prune_batch_kernel" if "prune_batch_kernel" in name
               else "expm" if "expm" in name else "memcpy" if "emcpy" in name or "->" in name else "other")
        groups[key] += us / 1e6
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "bench_joint_ancestors_kernels.txt"), "a") as f:
            f.write(prof.key_averages().table(sort_by="device_time_total", row_limit=30) + "\n")
    return groups


def run(lf, w, shape, reps, out_dir):
    V, W, bk, bg = make_sets(w, shape)
    pats = np.arange(w.S)
    part = lf.part
    new = lambda: part.batch_joint_ancestors(pats, V, w.pi, weights=W, branch_k=bk, branch_group=bg)  # noqa: E731
    with_site = lambda: part.batch_joint_ancestors(pats, V, w.pi, weights=W, branch_k=bk, branch_group=bg,  # noqa: E731
                                                   want_site=True)
    if W is None:
        site_call = lambda: part.batch_site_likelihoods(pats, V, w.pi, branch_group=bg)       # noqa: E731
    else:
        site_call = lambda: part.batch_site_mixture_likelihoods(pats, V, W, w.pi, branch_k=bk, branch_group=bg)  # noqa: E731
    st, jl = new()                                                      # warm-up
    st2, jl2, site = with_site()
    lnl = site_call()
    t_new, s_new = median_time(new, reps)
    t_site, s_site = median_time(site_call, reps)
    groups = profile(with_site, out_dir)
    return {"shape": shape, "sets": int(w.S), "internal_nodes": int(w.tree.n_internal), "states": int(w.D),
            "new_s": t_new, "new_spread_s": s_new, "new_sets_per_s": w.S / t_new,
            "site_call_s": t_site, "site_call_spread_s": s_site, "site_call_sets_per_s": w.S / t_site,
            "new_over_site_call": t_new / t_site, "kernel_s": groups,
            "joint_over_prune": groups["joint_ancestors_kernel"] / groups["prune_batch_kernel"],
            "site_equals_site_call": bool(np.array_equal(site, lnl)),
            "same_with_site": bool(np.array_equal(st, st2) and np.array_equal(jl, jl2)),
            "unresolved": int((st < 0).sum()), "finite_lnl": int(np.isfinite(jl).sum()),
            "sha256_states": hashlib.sha256(st.tobytes()).hexdigest()[:16],
            "sha256_lnl": hashlib.sha256(jl.tobytes()).hexdigest()[:16]}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reps", type=int, default=5)
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
        out["results"].append(run(lf, w, shape, args.reps, args.profile_dir))
    lf.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
