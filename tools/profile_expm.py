"""Where the expm stage of one resident evaluation goes, on the north-star workload of bench.py (200 taxa x 2000 codons,
MG94xREV, 4 omega classes, dense Q*t resident).  Warms up, then runs hb2_time_resident under torch.profiler with CUDA
activities and writes to the directory given by --out:
  trace.pt.trace.json  the raw trace
  expm_profile.json    per expm kernel: launches per evaluation and mean / min time; the gaps between consecutive
                       kernels of the stage and from its last kernel to the first pruning kernel; the stage's kernel span;
                       the card name and power limit read in the same run.
Run it in a process of its own: tracing slows the host, so its numbers are a breakdown, not a rate."""
import argparse
import json
import os
import statistics
import subprocess
import sys

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
    ap.add_argument("--out", required=True, metavar="DIR", help="output directory")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    import torch
    from torch.profiler import profile, ProfilerActivity
    from hyphy_b200 import synth, LikelihoodFunction
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import bench

    os.makedirs(args.out, exist_ok=True)
    torch.cuda.set_device(0)
    w = synth.codon_workload(bench.WORKLOAD["taxa"], bench.WORKLOAD["codons"], bench.WORKLOAD["classes"])
    lf = LikelihoodFunction(w, device=0)
    Qt = np.ascontiguousarray(w.Qt())
    for c in range(w.C):
        lf.part.set_matrices(c, lf.all_nodes, Qt[c])
    lf.part.time_resident(w.class_weights, w.pi, iters=args.warmup)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ms, stage, lnl = lf.part.time_resident(w.class_weights, w.pi, iters=args.iters)
        torch.cuda.synchronize()
    lf.close()
    trace = os.path.join(args.out, "trace.pt.trace.json")
    prof.export_chrome_trace(trace)

    kernels = sorted((e for e in json.load(open(trace))["traceEvents"] if e.get("cat") == "kernel"), key=lambda e: e["ts"])
    short = lambda e: e["name"].split("(")[0].split("<")[0].replace("void ", "").replace("hb2::", "")
    # one evaluation = a run of expm kernels followed by everything up to the next expm kernel
    evals, cur = [], None
    for e in kernels:
        is_expm = short(e).startswith("expm")
        if is_expm and (cur is None or not cur["expm_open"]):
            cur = {"expm": [], "rest": [], "expm_open": True}
            evals.append(cur)
        if cur is None:
            continue
        if is_expm and cur["expm_open"]:
            cur["expm"].append(e)
        else:
            cur["expm_open"] = False
            cur["rest"].append(e)
    evals = [v for v in evals if v["expm"] and v["rest"]]
    per_kernel, gaps, spans = {}, {}, []
    for v in evals:
        ex = v["expm"]
        for e in ex:
            per_kernel.setdefault(short(e), []).append(e["dur"])
        for a, b in zip(ex, ex[1:] + [v["rest"][0]]):
            key = f"{short(a)} -> {short(b)}"
            gaps.setdefault(key, []).append(b["ts"] - (a["ts"] + a["dur"]))
        spans.append(v["rest"][0]["ts"] - ex[0]["ts"])
    n = max(len(evals), 1)
    summ = lambda xs: {"mean_us": statistics.fmean(xs), "min_us": min(xs), "max_us": max(xs)}
    out = {"workload": bench.NAME, "evaluations_traced": len(evals),
           "kernels": {k: dict(summ(v), launches_per_eval=len(v) / n) for k, v in per_kernel.items()},
           "gaps": {k: summ(v) for k, v in gaps.items()},
           "expm_span_us": summ(spans) if spans else None,
           "expm_kernel_sum_us": sum(statistics.fmean(v) * len(v) / n for v in per_kernel.values()),
           "time_resident_stage_ms_under_profiler": {"expm": stage[0], "pruning": stage[1], "root": stage[2]},
           "lnL": lnl, **card()}
    json.dump(out, open(os.path.join(args.out, "expm_profile.json"), "w"), indent=1)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
