"""Site-level parametric bootstrap (FEL / MEME --resample N) on the north-star alignment (200 taxa x 2000 codons, MG94xREV),
one set per pattern, in the two site-model shapes of tools/bench_batch_sites.py:
  fel         one matrix per branch, tested / background branches as the group hint
  meme_third  K = 2 on a seeded third of the branches, one component elsewhere
For each shape it reports
  simulate    hb2_batch_site_simulate, N replicate columns of every set (N = --reps-list), as columns/s
  score       hb2_batch_column_likelihoods of one simulated replicate per set under the set's own values, as columns/s
  patterns    the column entry point fed the partition's own patterns against hb2_batch_site_likelihoods /
              hb2_batch_site_mixture_likelihoods on the same sets, calls alternated: both run the same pruning kernel, so
              the ratio is the cost of the column table
Every call is warmed up once, then timed with a host clock around the blocking call; the median of --repeat calls is
reported with the card's name and power limit read in the same run.  One JSON line on stdout."""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np  # noqa: E402

from hyphy_b200 import synth, LikelihoodFunction, engine  # noqa: E402
from bench_batch_sites import card, make_sets  # noqa: E402

SHAPES = ("fel", "meme_third")


def timed(call, repeat):
    call()                                                               # warm-up: buffers, modules
    times = []
    for _ in range(repeat):
        t0 = time.perf_counter()
        call()                                                           # returns after the stream is synchronised
        times.append(time.perf_counter() - t0)
    return float(np.median(times)), [min(times), max(times)]


def run(lf, w, shape, reps_list, repeat):
    V, W, bk, bg = make_sets(w, shape)
    part, S = lf.part, w.S
    out = {"shape": shape, "sets": int(S), "rows_per_set": int(V.shape[1]), "simulate": []}
    for n in reps_list:
        t, spread = timed(lambda: part.batch_site_simulate(V, w.pi, n, weights=W, branch_k=bk, branch_group=bg, seed=1), repeat)
        out["simulate"].append({"reps": n, "median_s": t, "spread_s": spread, "columns_per_s": S * n / t})
    leaf, _ = part.batch_site_simulate(V, w.pi, 1, weights=W, branch_k=bk, branch_group=bg, seed=2)
    cols = np.ascontiguousarray(leaf[:, 0])
    t, spread = timed(lambda: part.batch_column_likelihoods(cols, V, w.pi, weights=W, branch_k=bk, branch_group=bg), repeat)
    out["score"] = {"median_s": t, "spread_s": spread, "columns_per_s": S / t}
    # the partition's own patterns through both entry points, alternated call by call
    pats = np.arange(S)
    own = np.ascontiguousarray(w.leaf_states.T)
    if W is None:
        by_pattern = lambda: part.batch_site_likelihoods(pats, V, w.pi, branch_group=bg)               # noqa: E731
    else:
        by_pattern = lambda: part.batch_site_mixture_likelihoods(pats, V, W, w.pi, branch_k=bk, branch_group=bg)  # noqa: E731
    by_column = lambda: part.batch_column_likelihoods(own, V, w.pi, weights=W, branch_k=bk, branch_group=bg)      # noqa: E731
    same = bool(np.array_equal(by_pattern(), by_column()))
    tp, tc = [], []
    for _ in range(repeat):
        for call, acc in ((by_pattern, tp), (by_column, tc)):
            t0 = time.perf_counter()
            call()
            acc.append(time.perf_counter() - t0)
    out["patterns"] = {"identical": same, "pattern_median_s": float(np.median(tp)), "column_median_s": float(np.median(tc)),
                       "column_over_pattern": float(np.median(tc) / np.median(tp))}
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--repeat", type=int, default=5)
    ap.add_argument("--reps-list", default="20,100", help="replicates per set of the simulate lines")
    ap.add_argument("--shapes", default=",".join(SHAPES), help="comma-separated subset of " + ", ".join(SHAPES))
    args = ap.parse_args()
    if engine.device_count() < 1:
        sys.exit("no CUDA device: this benchmark measures the GPU and has nothing to fall back to")
    info = card()
    w = synth.codon_workload(200, 2000, 1)
    lf = LikelihoodFunction(w, flags=engine.FLAG_FORCE_FP64)
    lf.set_template()
    out = dict(info, workload=f"MG94xREV {w.tree.n_leaves}x2000, {w.S} patterns, {w.tree.n_branches} branches", results=[])
    for shape in args.shapes.split(","):
        out["results"].append(run(lf, w, shape, [int(x) for x in args.reps_list.split(",")], args.repeat))
    lf.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
