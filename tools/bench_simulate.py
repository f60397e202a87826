"""Throughput of hb2_simulate on the north-star tree and model of bench.py (200 taxa, MG94xREV, 4 omega classes, dense Q*t
handed over): `--reps` replicates of `--sites` sites each, one call per replicate (leaf states only, as a parametric
bootstrap consumes them).
  1. wall clock around the calls (host buffers, each call ends in a stream synchronise): simulated sites/s;
  2. a second pass under torch.profiler with CUDA activities (CUPTI activity records rather than CUDA events: the kernels
     run on the engine's own stream, which events recorded from Python cannot bracket): device time per replicate of
     sim_cdf_kernel and simulate_kernel, and of the device-to-host copies of the leaf states (the 4-byte read-back of
     the bad-row flag is left out by its size).
Prints one JSON object with the card name and power limit read in the same run; --out DIR also writes it and the trace."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402


def card():
    try:
        line = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in line.split(",")]
        return {"card": name, "power_limit": power, "sm_clock_max": clock}
    except (OSError, subprocess.SubprocessError, IndexError, ValueError):
        return {"card": None, "power_limit": None, "sm_clock_max": None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=100)
    ap.add_argument("--sites", type=int, default=2000)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default="", metavar="DIR", help="also write bench_simulate.json and the profiler trace here")
    args = ap.parse_args()
    import torch
    from torch.profiler import profile, ProfilerActivity
    from hyphy_b200 import synth, LikelihoodFunction
    import bench

    torch.cuda.set_device(0)
    w = synth.codon_workload(bench.WORKLOAD["taxa"], bench.WORKLOAD["codons"], bench.WORKLOAD["classes"])
    lf = LikelihoodFunction(w, device=0)
    lf.set_all_matrices()
    for k in range(args.warmup):
        lf.simulate(args.sites, seed=1000 + k)

    t0 = time.perf_counter()
    for r in range(args.reps):
        leaf, _, _ = lf.simulate(args.sites, seed=r)
    wall = time.perf_counter() - t0

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for r in range(args.reps):
            lf.simulate(args.sites, seed=r)
        torch.cuda.synchronize()
    lf.close()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
    trace = os.path.join(args.out or tempfile.gettempdir(), f"bench_simulate_{os.getpid()}.pt.trace.json")
    prof.export_chrome_trace(trace)
    events = json.load(open(trace))["traceEvents"]
    if not args.out:
        os.remove(trace)
    short = lambda e: e["name"].split("(")[0].split("<")[0].replace("void ", "").replace("hb2::", "")
    kern, d2h = {}, []
    for e in events:
        if e.get("cat") == "kernel" and short(e) in ("sim_cdf_kernel", "simulate_kernel"):
            kern.setdefault(short(e), []).append(e["dur"])
        elif e.get("cat") == "gpu_memcpy" and "DtoH" in e["name"] and e.get("args", {}).get("bytes", 0) > 64:
            d2h.append(e["dur"])
    per_rep = lambda xs: sum(xs) / args.reps
    ns = args.reps * args.sites
    out = {"workload": f"{bench.NAME}: tree and model, {args.reps} replicates x {args.sites} sites",
           "taxa": w.tree.n_leaves, "states": w.D, "classes": w.C,
           "simulated_sites_per_s": ns / wall, "wall_ms_per_replicate": wall / args.reps * 1e3,
           "kernel_us_per_replicate": {k: per_rep(v) for k, v in kern.items()},
           "kernel_launches_per_replicate": {k: len(v) / args.reps for k, v in kern.items()},
           "state_copy_us_per_replicate": per_rep(d2h), "state_copies_per_replicate": len(d2h) / args.reps,
           "state_bytes_per_replicate": w.tree.n_leaves * args.sites * 8,
           "cdf_table_bytes": w.C * w.tree.n_branches * w.D * 64 * 8, **card()}
    if args.out:
        json.dump(out, open(os.path.join(args.out, "bench_simulate.json"), "w"), indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
