"""hb2_batch_site_rates on two LEISR-shaped workloads (LEISR.bf:271-290, :420-444; relative_prot_rates.bf:160-192):
  nucleotide  synth.nucleotide_workload(256, 20000), HKY85 through its compiled template
  protein     synth.generic_workload(20, 128, 5000), a 20-state reversible model through its compiled template
each measured three ways:
  (a) grid    one set per pattern at each of LEISR's six start rates (0.01, 0.1, 0.5, 1, 2, 10): 6 S sets in one call
  (b) random  one set per pattern at its own random rate (one optimiser iteration over every site)
  (c) common  what the resident path can do: one common rate per call (compiled hand-over of every branch at that rate,
              then hb2_evaluate with per-pattern output), six calls, one per grid rate
Each is warmed up, then the median of --reps blocking calls is taken with a host clock; (a) and (b) report sets/s and
matrices/s (sets x branches), (c) patterns x rates per second.  A second pass under torch.profiler gives the device time
of expm_rates_kernel and prune_rates_kernel per call, and the algorithmic bytes of the P matrices written by the first
and read by the second over that time against the H100 SXM's 3.35 TB/s.  The card's name, power limit and SM clock are
read in the same run.  One JSON line on stdout; `sha256` fingerprints the log-likelihoods of the first call."""
import argparse
import hashlib
import json
import os
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from hyphy_b200 import synth, LikelihoodFunction, engine  # noqa: E402
from tools.bench_batch_sites import card  # noqa: E402

GRID = np.array([0.01, 0.1, 0.5, 1.0, 2.0, 10.0])        # LEISR.bf:420-444
HBM_BYTES_PER_S = 3.35e12                                 # H100 SXM data sheet
KERNELS = ("expm_rates_kernel", "prune_rates_kernel")


def workloads():
    return {"nucleotide": synth.nucleotide_workload(256, 20000), "protein": synth.generic_workload(20, 128, 5000)}


def pad(D):
    return next(p for p in (4, 8, 16, 24, 32) if D <= p)


def timed(call, reps):
    first = call()                                        # warm-up: workspace, modules
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        call()                                            # returns after the stream is synchronised
        times.append(time.perf_counter() - t0)
    return first, float(np.median(times)), [min(times), max(times)]


def calls(lf, w):
    S, vals = w.S, w.compiled_values()[0]
    rng = np.random.default_rng(1)
    pats = np.arange(S)
    grid_p, grid_r = np.tile(pats, len(GRID)), np.repeat(GRID, S)
    rand_r = 10.0 ** rng.uniform(-2, 1, S)

    def common():
        out = np.empty((len(GRID), S))
        for k, r in enumerate(GRID):
            lf.part.set_matrices_compiled(0, lf.all_nodes, vals * r)
            _, sl, ss = lf.part.evaluate(0, w.pi, want_sites=True)
            out[k] = np.log(sl) - 64.0 * np.log(2.0) * ss
        return out

    return {"grid": (lambda: lf.part.batch_site_rates(grid_p, grid_r, w.pi), len(grid_p)),
            "random": (lambda: lf.part.batch_site_rates(pats, rand_r, w.pi), S),
            "common": (common, len(GRID) * S)}


def profile_kernels(fn, reps, out_dir):
    import torch
    from torch.profiler import profile, ProfilerActivity
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    trace = os.path.join(out_dir or tempfile.gettempdir(), f"bench_site_rates_{os.getpid()}.pt.trace.json")
    prof.export_chrome_trace(trace)
    events = json.load(open(trace))["traceEvents"]
    os.remove(trace)
    short = lambda e: e["name"].split("(")[0].split("<")[0].replace("void ", "").replace("hb2::", "")   # noqa: E731
    us = {k: 0.0 for k in KERNELS}
    for e in events:
        if e.get("cat") == "kernel" and short(e) in us:
            us[short(e)] += e["dur"]
    return {k: v / reps for k, v in us.items()}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default="", metavar="DIR", help="also write bench_site_rates.json here")
    args = ap.parse_args()
    if engine.device_count() < 1:
        sys.exit("no CUDA device: this benchmark measures the GPU and has nothing to fall back to")
    out = dict(card(), results=[])
    for name, w in workloads().items():
        lf = LikelihoodFunction(w, flags=engine.FLAG_FORCE_FP64)
        lf.set_template()
        lf.set_all_compiled()
        B, Dp = w.tree.n_branches, pad(w.D)
        res = {"workload": name, "taxa": w.tree.n_leaves, "states": w.D, "patterns": int(w.S), "branches": B}
        for how, (fn, n) in calls(lf, w).items():
            first, t, spread = timed(fn, args.reps)
            r = {"median_s": t, "spread_s": spread, "sets_per_s": n / t,
                 "finite": int(np.isfinite(first).sum()), "sha256": hashlib.sha256(np.ascontiguousarray(first).tobytes()).hexdigest()[:16]}
            if how != "common":
                r["matrices_per_s"] = n * B / t
                us = profile_kernels(fn, args.reps, args.out)
                p_bytes = 2.0 * n * B * Dp * Dp * 8                # P area written by the exponential, read by the pruning
                dev_s = sum(us.values()) * 1e-6
                r.update(kernel_us_per_call=us, p_bytes_per_call=p_bytes, p_bytes_per_s=p_bytes / dev_s,
                         share_of_hbm_peak=p_bytes / dev_s / HBM_BYTES_PER_S)
            res[how] = r
        lf.close()
        out["results"].append(res)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        json.dump(out, open(os.path.join(args.out, "bench_site_rates.json"), "w"), indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
