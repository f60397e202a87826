"""Batched one-pattern likelihoods on the north-star alignment (200 taxa x 2000 codons, MG94xREV), one set per pattern,
shaped like the site phases of FEL and MEME:
  fel        one matrix per branch (hb2_batch_site_likelihoods), tested / background branches as the group hint
  meme_all   K = 2 components on every branch (hb2_batch_site_mixture_likelihoods)
  meme_third K = 2 on a seeded third of the branches, one component elsewhere, tested / background as the group hint
Each shape is warmed up with one call of the same size, then timed with a host clock around the blocking call; the median
of --reps calls is reported as sets/s and component matrices exponentiated per second, with the card's name and power
limit read in the same run.  One JSON line on stdout; `sha256` fingerprints the log-likelihoods of the first call."""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from hyphy_b200 import synth, LikelihoodFunction, engine  # noqa: E402

SHAPES = ("fel", "meme_all", "meme_third")


def card():
    try:
        line = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in line.split(",")]
        return {"card": name, "power_limit": power, "sm_clock_max": clock}
    except (OSError, subprocess.SubprocessError, IndexError, ValueError):
        return {"card": None, "power_limit": None, "sm_clock_max": None}


def with_omega(w, omega):
    return synth.Workload(w.name, w.tree, w.D, w.pi, [synth.mg94_rev_Q(omega)], np.array([1.0]), w.leaf_states, w.ambig,
                          w.pattern_freq, w.site_to_pattern, None, dict(w.meta, omegas=[omega]))


def make_sets(w, shape, seed=1):
    """(formula values, weights or None, branch_k or None, branch_group) of one set per pattern."""
    rng = np.random.default_rng(seed)
    nb, S = w.tree.n_branches, w.S
    unit = with_omega(w, 1.0).compiled_values()[0]                      # [B, nF] at omega = 1
    nonsyn = ~np.isclose(with_omega(w, 2.0).compiled_values()[0][0], unit[0])
    tested = np.zeros(nb, dtype=bool)
    tested[rng.choice(nb, nb // 3, replace=False)] = True
    alpha = rng.uniform(0.5, 2.0, S)
    betas = np.sort(rng.uniform(0.0, 4.0, (S, 3)), axis=1)             # column 0: background; 1, 2: the two components
    w0 = rng.uniform(0.5, 0.95, S)
    if shape == "fel":
        col = np.where(tested, 2, 0)
        row_branch, row_w = np.arange(nb), None
    else:
        branch_k = np.full(nb, 2) if shape == "meme_all" else np.where(tested, 2, 1)
        row_branch = np.repeat(np.arange(nb), branch_k)
        first = np.concatenate([[0], np.cumsum(branch_k)[:-1]])
        comp = np.arange(len(row_branch)) - first[row_branch]              # component index of each row
        col = np.where(branch_k[row_branch] == 2, 1 + comp, 0)
        row_w = np.where(col == 0, 1.0, np.where(col == 1, w0[:, None], 1.0 - w0[:, None]))
    V = unit[row_branch][None] * np.where(nonsyn[None, None, :], betas[:, col][:, :, None], alpha[:, None, None])
    bg = None if shape == "meme_all" else tested.astype(np.int64)
    bk = None if shape == "fel" else branch_k.astype(np.int64)
    return np.ascontiguousarray(V), row_w, bk, bg


def run(lf, w, shape, reps):
    V, W, bk, bg = make_sets(w, shape)
    pats = np.arange(w.S)
    if W is None:
        call = lambda: lf.part.batch_site_likelihoods(pats, V, w.pi, branch_group=bg)          # noqa: E731
    else:
        call = lambda: lf.part.batch_site_mixture_likelihoods(pats, V, W, w.pi, branch_k=bk, branch_group=bg)   # noqa: E731
    first = call()                                                      # warm-up: buffers, modules
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        call()                                                          # returns after the stream is synchronised
        times.append(time.perf_counter() - t0)
    t = float(np.median(times))
    rows = V.shape[1]
    return {"shape": shape, "sets": int(w.S), "rows_per_set": int(rows), "median_s": t, "spread_s": [min(times), max(times)],
            "sets_per_s": w.S / t, "matrices_per_s": w.S * rows / t, "finite": int(np.isfinite(first).sum()),
            "sha256": hashlib.sha256(first.tobytes()).hexdigest()[:16]}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reps", type=int, default=5)
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
        out["results"].append(run(lf, w, shape, args.reps))
    lf.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
