#!/usr/bin/env python
"""bench.py -- LF evaluations/second on the north-star workload (200 taxa x 2000 codons, MG94xREV, 4 omega classes).

    python bench.py [--gpus N] [--steps K] [--warmup W] [--impl reference] [--dump-outputs DIR]
    N>1: python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 ... bench.py --gpus N ...

A "step" is ONE full likelihood-function evaluation: every one of the B*C rate matrices handed over, exponentiated,
the whole tree pruned for all patterns and classes, root reduction, one fp64 lnL back.
  value : evaluations/s with the inputs already resident in HBM (device time, CUDA events on the engine's stream,
          K steps, max over ranks).
  e2e   : the same through the public C-ABI call sequence a host makes per evaluation (hb2_set_matrices_compiled for
          every class + hb2_evaluate_classes) with HOST buffers: the H2D copy of that step's formula values and the D2H
          read of lnL are inside the timed region.  e2e_dense is the same with dense D*D rate matrices
          (hb2_set_matrices_packed), i.e. without the compiled-template hand-over.
Multi-GPU (strong scaling of one alignment): ranks form (pattern shards) x (class groups) -- rate classes first, so no
rank exponentiates another group's matrices, patterns for the remaining factor (hyphy_b200/sharding.py); one exchange
per evaluation on the engine's own NCCL communicator.
The oracle / reference binary under oracle/ is used only for cpu_baseline and --impl reference.
--dump-outputs DIR: after the timed steps, the outputs of the last timed evaluation of each timed path as DIR/<name>.npy
(float64): the lnL values, and the per-pattern log-likelihoods and scaling exponents of the resident path recomputed
from the same resident state.  Inputs are seeded, so two builds run with the same arguments can be compared output by output.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

WORKLOAD = dict(taxa=200, codons=2000, classes=4)
NAME = "MG94xREV 200 taxa x 2000 codons, 4 omega classes (synthetic, seed 20260924)"
METRIC = "LF evals/sec, 200-taxon x 2000-codon MG94xREV 4 omega-cats"


def peaks():
    try:
        return json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))), "measured"
    except Exception:
        return {"hbm_gbs": 3350.0, "bf16_tflops": 989.0}, "fallback: H100 SXM data sheet"


class ClockSampler:
    """nvidia-smi sampling DURING the timed region: SM clock and throttle reasons."""
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, device):
        self.path = tempfile.mktemp(prefix="hb2clk_", suffix=".csv")
        self.proc = None
        self.device = device

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.device), f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                                          "-lms", "100"], stdout=open(self.path, "w"), stderr=subprocess.DEVNULL)
        except Exception:
            self.proc = None

    def wait_first_sample(self, timeout=5.0):
        t0 = time.time()
        while time.time() - t0 < timeout:
            try:
                if os.path.getsize(self.path) > 0:
                    return True
            except OSError:
                pass
            time.sleep(0.02)
        return False

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.15)
        self.proc.terminate()
        try:
            self.proc.wait(timeout=5)
        except Exception:
            self.proc.kill()
        sm, mx, reasons = [], [], set()
        for line in open(self.path):
            f = [x.strip() for x in line.split(",")]
            if len(f) < 9:
                continue
            try:
                sm.append(float(f[1])); mx.append(float(f[2]))
            except ValueError:
                continue
            for nm, v in zip(["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"], f[5:9]):
                if v.lower().startswith("active"):
                    reasons.add(nm)
        try:
            os.unlink(self.path)
        except OSError:
            pass
        if not sm:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["no samples"]}
        return {"sm_mhz": statistics.median(sm), "sm_max_mhz": max(mx), "reasons": sorted(reasons), "samples": len(sm)}


def algorithmic_work(w, S, word=8):
    """SURVEY.md §8(d) per-evaluation algorithmic work for S patterns (all classes); `word` = bytes per stored
    conditional (8 on the fp64 path, 4 on the tensor-core path)."""
    L, I, D, C = w.tree.n_leaves, w.tree.n_internal, w.D, w.C
    B = L + I - 1
    flops = C * ((I - 1) * S * 2 * D * D + (L + B) * S * D + 2 * S * D)
    byts = C * ((2 * I - 1) * S * D * word + B * D * D * 8 + L * S)
    expm_flops = C * B * 5 * 2 * 64 ** 3         # this engine: ~5.0 products of 64^3 per matrix on this stream (DESIGN §4.1)
    return flops, byts, expm_flops


def cpu_baseline_full(steps, warmup, threads, probe=True):
    """Reference HYPHYMP (oracle/_ref/hyphy) on the FULL stated workload (200 x 2000 x 4 classes): `steps` timed full
    evaluations after `warmup`, each perturbing one global parameter so every matrix is re-exponentiated (SURVEY §8d).
    No sub-sampling and no extrapolation: the number is evaluations/s of the same config the GPU arm runs."""
    from hyphy_b200 import synth
    from oracle import ref_harness as rh, port
    w = synth.codon_workload(WORKLOAD["taxa"], WORKLOAD["codons"], WORKLOAD["classes"])
    if rh.have_reference():
        # the reference tunes its own thread count (BenchmarkThreads, likefunc.cpp:219); give it the same courtesy:
        # a short probe over a few counts (2 full-size evaluations each), then the timed run at the best one
        best = threads
        probe_rates = {}
        if probe:
            cands = sorted({t for t in (8, 16, 32, 64, threads) if t <= threads})
            best, best_rate = cands[0], 0.0
            for t in cands:
                pr = rh.run_reference(w, n_evals=2, threads=t, per_site=False, n_warm=1)
                probe_rates[t] = 2 / pr["loop_seconds"]
                if probe_rates[t] > best_rate:
                    best, best_rate = t, probe_rates[t]
        r = rh.run_reference(w, n_evals=steps, threads=best, per_site=False, n_warm=warmup)
        rate = steps / r["loop_seconds"]
        kind, cores, lnl = "reference", best, r["lnL"]
    else:
        port.lnl(w)
        n = max(1, min(steps, 2))
        t0 = time.perf_counter()
        for _ in range(n):
            lnl, _ = port.lnl(w)
        rate = n / (time.perf_counter() - t0)
        kind, cores, probe_rates = "port", 1, {}
    return dict(kind=kind, cores=cores, rate=rate, S=w.S, lnl=lnl, probe=probe_rates,
                sample=f"full workload: {WORKLOAD['taxa']} taxa x {WORKLOAD['codons']} codons x {WORKLOAD['classes']} classes "
                       f"(S={w.S} patterns), {steps} full evaluations after {warmup} warm-up, no extrapolation")


def config_dict(S, B, D, C):
    """Identical for both arms (the driver compares them): the workload and nothing implementation-specific."""
    return {"workload": NAME, "taxa": WORKLOAD["taxa"], "codons": WORKLOAD["codons"], "patterns": S, "branches": B, "states": D,
            "classes": C, "l2": "inputs larger than L2 (830 MB of conditionals per evaluation)"}


def run_reference_arm(args, rank):
    """--impl reference: the unmodified reference binary (HYPHYMP, OpenMP + AVX2) on the box's host cores, same config."""
    if rank != 0:
        return
    threads = os.cpu_count() or 1
    t0 = time.time()
    cb = cpu_baseline_full(args.steps, args.warmup, threads)
    value = cb["rate"]
    L = WORKLOAD["taxa"]
    line = {"impl": "reference", "metric": METRIC, "value": value, "unit": "evals/s", "n_gpus": args.gpus, "steps": args.steps,
            "warmup": args.warmup, "ms_per_step": 1000.0 / value, "higher_is_better": True, "scaling": "strong",
            "vs_baseline": None, "dtype": "f64", "data": "synthetic",
            "config": config_dict(cb["S"], 2 * L - 3, 61, WORKLOAD["classes"]),
            "layout": "host cores (OpenMP), no GPU",
            "cpu_baseline": {"value": value, "unit": "evals/s", "cores": cb["cores"], "kind": cb["kind"], "sample": cb["sample"],
                             "thread_probe_evals_per_s": cb["probe"]},
            "e2e": {"value": value, "unit": "evals/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
            "gpu_launches": 0, "lnL": cb["lnl"], "wall_s": time.time() - t0}
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-host", action="store_true", help="skip the patched-HyPhy end-to-end leg")
    ap.add_argument("--no-c5", action="store_true", help="skip the extra 500 x 5000 x 4 line")
    ap.add_argument("--no-small", action="store_true", help="skip the nucleotide / protein extra lines")
    ap.add_argument("--fp64", action="store_true", help="force the fp64 pruning kernels (HB2_FLAG_FORCE_FP64)")
    ap.add_argument("--class-groups", type=int, default=0, help="multi-GPU: force this many class groups (default: as many as divide both)")
    ap.add_argument("--no-class-groups", action="store_true", help="multi-GPU: shard patterns only (every rank exponentiates every class)")
    ap.add_argument("--emulate-shard", default="", help="debug: R/W -> run rank R's pattern shard of a W-rank job on one GPU, no collectives")
    ap.add_argument("--dump-outputs", default="", metavar="DIR", help="write the last timed evaluation's outputs as DIR/<name>.npy")
    args = ap.parse_args()
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    if args.impl == "reference":
        run_reference_arm(args, rank)
        return
    assert args.warmup >= 3, "timing rules: at least 3 warm-up steps"
    assert world == args.gpus, f"--gpus {args.gpus} but WORLD_SIZE={world} (launch with torch.distributed.run)"

    import torch
    from hyphy_b200 import synth, LikelihoodFunction, Partition
    torch.cuda.set_device(local_rank)
    dist = None
    if world > 1:
        # control plane (barriers, id exchange, max-over-ranks of the timings) over gloo; the DATA path -- the per-evaluation
        # exchange of class partials / partial log-likelihoods -- is the engine's own NCCL communicator (hb2_comm_init) on
        # the engine's stream, so no torch-owned NCCL communicator is needed in this process.
        import torch.distributed as dist
        dist.init_process_group("gloo")

    w = synth.codon_workload(WORKLOAD["taxa"], WORKLOAD["codons"], WORKLOAD["classes"])
    S = w.S
    from hyphy_b200.sharding import shard_bounds, exchange_unique_id, layout
    # (pattern shards) x (class groups): classes first (no replicated expm inside a shard), patterns for the rest (SURVEY §8e)
    lay = layout(world, rank, w.C, S)
    if args.class_groups > 0:                      # override: G class groups x world/G pattern shards
        G = args.class_groups
        assert w.C % G == 0 and world % G == 0, "--class-groups must divide both the classes and the ranks"
        lo_, hi_ = shard_bounds(S, world // G, rank // G)
        per = w.C // G
        lay = {"groups": G, "group": rank % G, "shards": world // G, "shard": rank // G, "patterns": (lo_, hi_), "classes": (rank % G * per, (rank % G + 1) * per)}
    if args.no_class_groups:
        lay = {"groups": 1, "group": 0, "shards": world, "shard": rank, "patterns": shard_bounds(S, world, rank), "classes": (0, w.C)}
    lo, hi = lay["patterns"]
    if args.emulate_shard:
        er, ew = (int(x) for x in args.emulate_shard.split("/"))
        lo, hi = shard_bounds(S, ew, er)
    lf = LikelihoodFunction(w, device=local_rank, flags=1 if args.fp64 else 0,
                            pattern_slice=slice(lo, hi) if (world > 1 or args.emulate_shard) else None)
    if world > 1:
        lf.part.comm_init(world, rank, exchange_unique_id(dist, rank, Partition.comm_unique_id))
        if lay["groups"] > 1:
            lf.part.comm_class_groups(lay["groups"])

    def barrier():
        if dist is not None:
            dist.barrier()
        torch.cuda.synchronize()

    def max_over_ranks(x):
        if dist is None:
            return x
        t = torch.tensor([x], dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    # per-step host inputs: one global parameter moved => every matrix changes (SURVEY §8d evaluation stream)
    n_variants = 4
    Qts = [np.ascontiguousarray(w.Qt(perturb=1e-4 * k)) for k in range(n_variants)]
    pinned = []
    for q in Qts:                                   # the host's matrices live in pinned memory
        t = torch.from_numpy(q).pin_memory()
        pinned.append(t)
    Qts = [t.numpy() for t in pinned]

    lf.set_template()                                # static half of the compiled model matrix, once
    Vs = [torch.from_numpy(np.ascontiguousarray(w.compiled_values(perturb=1e-4 * k))).pin_memory().numpy() for k in range(n_variants)]

    def e2e_step(k):
        lf.set_all_compiled(Vs[k % n_variants])
        return lf.compute()

    def e2e_dense_step(k):
        q = Qts[k % n_variants]
        for c in range(w.C):
            lf.part.set_matrices(c, lf.all_nodes, q[c])
        return lf.compute()

    last = {}

    def timed(step):
        for k in range(args.warmup):
            step(k)
        barrier()
        t0 = time.perf_counter()
        for k in range(args.steps):
            last[step.__name__] = step(k)
        barrier()
        return max_over_ranks((time.perf_counter() - t0) * 1e3 / args.steps)

    lnl0 = e2e_step(0)                              # also the first (whole-tree) evaluation
    lnl_dense = e2e_dense_step(0)
    # ---- e2e: public API with host buffers ---------------------------------------------------------
    e2e_dense_ms = timed(e2e_dense_step)
    e2e_ms = timed(e2e_step)
    # where the host-side part of an end-to-end step goes (separate untimed-for-the-record loop, wall clock on this rank)
    t_set = t_eval = 0.0
    for k in range(args.steps):
        t0 = time.perf_counter()
        lf.set_all_compiled(Vs[k % n_variants])
        t1 = time.perf_counter()
        lf.compute()
        t_eval += time.perf_counter() - t1
        t_set += t1 - t0
    e2e_split = {"set_matrices_ms": t_set * 1e3 / args.steps, "evaluate_ms": t_eval * 1e3 / args.steps}
    # ---- resident: device time by CUDA events on the engine's stream ---------------------------------
    lf.part.set_matrices(0, lf.all_nodes, Qts[0][0])
    for c in range(1, w.C):
        lf.part.set_matrices(c, lf.all_nodes, Qts[0][c])
    lf.part.time_resident(w.class_weights, w.pi, iters=args.warmup)
    sampler = ClockSampler(local_rank)
    sampler.start()
    sampler.wait_first_sample()
    launches0 = lf.part.launch_count
    barrier()
    ms, stage, lnl_res = lf.part.time_resident(w.class_weights, w.pi, iters=args.steps)
    barrier()
    launches = lf.part.launch_count - launches0
    dump = {}
    if args.dump_outputs:
        # per-pattern outputs of the resident state the timed loop evaluated (same matrices, nothing re-staged)
        lnl_sites, site_l, site_s = lf.compute(want_sites=True)
        dump = {"lnL_resident": np.array([lnl_res]), "lnL_e2e": np.array([last["e2e_step"]]),
                "lnL_e2e_dense": np.array([last["e2e_dense_step"]]), "lnL_sites_eval": np.array([lnl_sites]),
                "site_lnL": np.asarray(site_l, dtype=np.float64), "site_scale": np.asarray(site_s, dtype=np.float64)}
    # the timed region is a few tens of ms; keep the identical load running ~1 s so nvidia-smi (100 ms period) sees it.
    # The repeat count is derived from the rank-reduced time so every rank issues the same number of all-reduces.
    extra = int(min(200, max(1, round(1000.0 / max(max_over_ranks(ms) * args.steps, 1e-3)))))
    for _ in range(extra):
        lf.part.time_resident(w.class_weights, w.pi, iters=args.steps)
    clocks = sampler.stop()
    tc_mode = lf.part.precision_mode == 1
    prune_kernel = lf.part.pruning_kernel
    root_path = "peer" if os.environ.get("HB2_PEER_XCHG", "1") != "0" else "nccl"
    stage_launches = [int(x) for x in lf.part.stage_launches]
    ms = max_over_ranks(ms)
    stage = [max_over_ranks(float(s)) for s in stage]
    lf.close()

    # ---- extra line: BASELINE.json configs[4] (c5: 500 taxa x 5000 codons x 4 classes, 5.2 GB of conditionals), the size at
    #      which sharding one alignment over the box pays; same measurement as `value` (resident, device time, max over ranks)
    c5 = None
    if not args.no_c5:
        w5 = synth.codon_workload(500, 5000, 4)
        lay5 = layout(world, rank, w5.C, w5.S)
        if args.no_class_groups:
            lay5 = {"groups": 1, "group": 0, "shards": world, "shard": rank, "patterns": shard_bounds(w5.S, world, rank), "classes": (0, w5.C)}
        lo5, hi5 = lay5["patterns"]
        lf5 = LikelihoodFunction(w5, device=local_rank, flags=1 if args.fp64 else 0, pattern_slice=slice(lo5, hi5) if world > 1 else None)
        if world > 1:
            lf5.part.comm_init(world, rank, exchange_unique_id(dist, rank, Partition.comm_unique_id))
            if lay5["groups"] > 1:
                lf5.part.comm_class_groups(lay5["groups"])
        lf5.set_template()
        lf5.set_all_compiled()
        lnl5 = lf5.compute()
        lf5.part.time_resident(w5.class_weights, w5.pi, iters=3)
        barrier()
        ms5, stage5, lnl5r = lf5.part.time_resident(w5.class_weights, w5.pi, iters=args.steps)
        barrier()
        ms5 = max_over_ranks(ms5)
        stage5 = [max_over_ranks(float(x)) for x in stage5]
        lf5.close()
        golden5 = -1160063.8295306289                 # unmodified reference binary (tests/golden/c5_mg94_500x5000_c4.npz)
        dump["lnL_c5_resident"] = np.array([lnl5r])
        c5 = {"workload": "MG94xREV 500 taxa x 5000 codons, 4 omega classes (BASELINE.json configs[4])", "patterns": w5.S,
              "value": 1000.0 / ms5, "unit": "evals/s", "ms_per_step": ms5, "stage_ms": {"expm": stage5[0], "pruning": stage5[1], "root": stage5[2]},
              "layout": f"patterns/{lay5['shards']} x classes/{lay5['groups']}", "lnL": lnl5, "lnL_reference": golden5,
              "rel_err": abs(lnl5 - golden5) / abs(golden5)}

    # ---- extra lines: the register kernels of the nucleotide (4 states) and protein (20 states) paths, HBM-bound by SURVEY §8d:
    #      achieved algorithmic GB/s of the pruning pass against the measured copy bandwidth (same numbers as tools/bench_small.py)
    small = None
    if world == 1 and not args.no_small:
        small = {}
        for key, wk in (("nucleotide_d4_256x200000", lambda: synth.nucleotide_workload(256, 200000, mean_t=0.1)),
                        ("protein_d20_128x20000_c4", lambda: synth.generic_workload(20, 128, 20000, 4, mean_t=0.1))):
            ws = wk()
            lfs = LikelihoodFunction(ws, device=local_rank)
            lfs.set_template()
            lfs.set_all_compiled()
            lfs.compute()
            lfs.part.time_resident(ws.class_weights, ws.pi, iters=3)
            mss, sts, lnls = lfs.part.time_resident(ws.class_weights, ws.pi, iters=args.steps)
            dump[f"lnL_{key}_resident"] = np.array([lnls])
            kern = lfs.part.pruning_kernel
            lfs.close()
            Ls, Is, Ss, Cs = ws.tree.n_leaves, ws.tree.n_internal, ws.S, ws.C
            Dps = 4 if ws.D <= 4 else (ws.D + 7) // 8 * 8
            bys = Cs * ((2 * Is - 1) * Ss * Dps * 8 + (2 * Is - 1) * Ss * 4 + Ls * Ss * 4)
            pk_, _k = peaks()
            small[key] = {"kernel": kern, "patterns": Ss, "ms_per_eval": mss, "pruning_ms": float(sts[1]), "algorithmic_bytes": bys,
                          "achieved_gbs": bys / (float(sts[1]) * 1e-3) / 1e9, "frac_of_hbm_peak": bys / (float(sts[1]) * 1e-3) / 1e9 / pk_["hbm_gbs"], "lnL": lnls}

    if rank == 0:
        pk, pk_kind = peaks()
        flops, byts, expm_flops = algorithmic_work(w, S, 4 if tc_mode else 8)
        # dominant kernel: the fused pruning pass; name and launches per evaluation come from the engine itself
        prune_launches = stage_launches[1]
        prune_ms = stage[1]
        achieved_gbs = (byts / world) / (prune_ms * 1e-3) / 1e9
        kname = {"prune64_tc_walk2_kernel": "prune64_tc_walk2_kernel (wgmma 3xTF32 fused pruning pass, whole tree in one launch, two threads per pattern)",
                 "prune64_tc_walk_kernel": "prune64_tc_walk_kernel (wgmma 3xTF32 fused pruning pass, whole tree in one launch)",
                 "prune64_tc_kernel": "prune64_tc_kernel (wgmma 3xTF32 fused pruning update, one launch per tree level)",
                 "prune64_kernel": "prune64_kernel (fp64 fused pruning update, one launch per tree level)"}.get(prune_kernel, prune_kernel)
        roofline = {"kernel": kname, "bound": "hbm",
                    "achieved": achieved_gbs, "peak": pk["hbm_gbs"], "unit": "GB/s", "frac": achieved_gbs / pk["hbm_gbs"],
                    "peak_source": f"MEASURED_PEAKS.json ({pk_kind})",
                    "launches_per_eval": prune_launches, "stage_launches_per_eval": {"expm": stage_launches[0], "pruning": stage_launches[1], "root": stage_launches[2]}, "avg_launch_ms": prune_ms / max(prune_launches, 1),
                    "algorithmic_bytes_per_eval": byts, "algorithmic_flops_per_eval": flops,
                    "tflops_pruning": (flops / world) / (prune_ms * 1e-3) / 1e12,
                    "tensor_frac_of_tf32_peak": ((flops / world) / (prune_ms * 1e-3) / 1e12) / (pk["bf16_tflops"] / 2) if tc_mode else None,
                    "fp64_tflops_expm": expm_flops / (stage[0] * 1e-3) / 1e12 if stage[0] > 0 else None,
                    "stage_ms": {"expm": stage[0], "pruning": stage[1], "root": stage[2]}}
        nF = w.compiled_template()[2]
        h2d = int(w.C * w.tree.n_branches * nF * 8 + w.C * w.tree.n_branches * 4 + (64 + w.C) * 8 + w.tree.n_internal * 4)
        h2d_dense = int(w.C * w.tree.n_branches * w.D * w.D * 8 + w.C * w.tree.n_branches * 4 + (64 + w.C) * 8 + w.tree.n_internal * 4)
        line = {"metric": METRIC, "value": 1000.0 / ms, "unit": "evals/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
                "ms_per_step": ms, "higher_is_better": True, "scaling": "strong", "vs_baseline": None,
                "dtype": "tf32x3 (wgmma, fp32 accumulate) pruning + f64 expm/root" if tc_mode else "f64",
                "data": "synthetic",
                "config": config_dict(S, w.tree.n_branches, w.D, w.C),
                "layout": f"patterns/{lay['shards']} x classes/{lay['groups']}",
                "e2e": {"value": 1000.0 / e2e_ms, "unit": "evals/s", "ms_per_step": e2e_ms, "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": 12,
                        "api": "hb2_set_matrices_compiled x C + hb2_evaluate_classes", "host_split": e2e_split},
                "e2e_dense": {"value": 1000.0 / e2e_dense_ms, "unit": "evals/s", "ms_per_step": e2e_dense_ms, "h2d_bytes_per_step": h2d_dense,
                              "d2h_bytes_per_step": 12, "api": "hb2_set_matrices_packed x C + hb2_evaluate_classes", "lnL": lnl_dense},
                "gpu_launches": int(launches), "clocks": clocks, "roofline": roofline, "lnL": lnl0, "lnL_resident": lnl_res,
                "lnL_reference": -205416.12461664603, "root_exchange": root_path if world > 1 else None, "c5": c5, "small_states": small}
        # the same evaluation stream through the PATCHED HyPhy binary (oracle/_ref/host/hyphy: the reference's HBL interpreter,
        # formula evaluation and DetermineNodesForUpdate on the host, everything below ComputeBlock on the engine):
        # wall-clock evaluations/s of `LFCompute` as a user of the reference would see them
        host_bin = os.path.join(ROOT, "oracle", "_ref", "host", "hyphy")
        if world == 1 and not args.no_host and os.path.isfile(host_bin):
            try:
                from oracle import ref_harness as rh
                hr = rh.run_reference(w, n_evals=args.steps, n_warm=args.warmup, per_site=False, binary=host_bin,
                                      env_extra={"HYPHY_B200_VERBOSE": "1", "HYPHY_B200_DEVICE": str(local_rank), "HYPHY_B200_TC": "1"})
                line["host_e2e"] = {"value": args.steps / hr["loop_seconds"], "unit": "evals/s", "lnL": hr["lnL"],
                                    "api": "patched HyPhy binary: HBL LFCompute -> _LikelihoodFunction::ComputeBlock -> hb2_hooks -> C ABI (dense Q*t hand-over)",
                                    "engine": hr["engine"][-2:]}
            except Exception as e:
                line["host_e2e"] = {"value": None, "error": repr(e)}
        if not args.no_cpu_baseline and world == 1:
            try:
                threads = os.cpu_count() or 1
                cb = cpu_baseline_full(6, 1, threads)
                line["cpu_baseline"] = {"value": cb["rate"], "unit": "evals/s", "cores": cb["cores"], "kind": cb["kind"], "sample": cb["sample"],
                                        "lnL": cb["lnl"]}
            except Exception as e:                   # the baseline is a report, never a reason to lose the bench line
                line["cpu_baseline"] = {"value": None, "unit": "evals/s", "cores": 0, "kind": "unavailable", "sample": repr(e)}
        print(json.dumps(line), flush=True)
    if args.dump_outputs:
        os.makedirs(args.dump_outputs, exist_ok=True)
        suffix = f"_rank{rank}" if world > 1 else ""
        for name, arr in dump.items():
            np.save(os.path.join(args.dump_outputs, name + suffix + ".npy"), np.ascontiguousarray(arr, dtype=np.float64))
    if dist is not None:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
