"""Worker of tests/test_multigpu.py (one process per GPU, launched by torch.distributed.run): evaluates a golden case on
`world` GPUs in the pattern-shard layout and in the (pattern shards) x (class groups) layout through the C ABI -- the
engine's own NCCL communicator carries the per-evaluation exchange -- and checks lnL and the shard's per-pattern outputs
against the unmodified reference binary's fixture."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


ZERO_WEIGHT_CASE = "class_groups_zero_weight"


def zero_weight_class_groups(world, rank, local, dist):
    """Two class groups, weights (0, 1): group 0 holds an identity class more than 1000 bits above group 1's uniform-row
    class on every pattern.  The weight-0 class takes no part, so lnL is class 1's alone, D^-leaves per pattern.
    Tolerances as on one GPU (class_merge_cases.tolerances: the tensor path's per-pattern bound grows with the tree)."""
    import math
    from hyphy_b200 import LikelihoodFunction, Partition, engine
    from hyphy_b200.sharding import shard_bounds, exchange_unique_id
    from tests import class_merge_cases as cm
    name = "d61_identity_uniform"
    D, n_leaves = cm.GAP_CASES[name][:2]
    w, P = cm.gap_case(name, weights=(0.0, 1.0))
    shards = world // 2
    lo, hi = shard_bounds(w.S, shards, rank // 2)
    want_site = -n_leaves * math.log(D)
    want = float(w.pattern_freq.sum()) * want_site
    out = []
    for flags, mode in ((engine.FLAG_FORCE_FP64, "fp64"), (engine.FLAG_DEFAULT, "tc")):
        rtol, atol = cm.tolerances(w, mode)
        lf = LikelihoodFunction(w, device=local, flags=flags, pattern_slice=slice(lo, hi))
        lf.part.comm_init(world, rank, exchange_unique_id(dist, rank, Partition.comm_unique_id))
        lf.part.comm_class_groups(2)
        for c in range(w.C):
            lf.part.set_matrices(c, lf.all_nodes, P[c], engine.MATRIX_TRANS)
        lnl, sl, ss = lf.compute(want_sites=True)
        lf.close()
        err = float(np.abs(np.log(sl) - 64.0 * np.log(2.0) * ss - want_site).max())
        ok = math.isfinite(lnl) and abs(lnl - want) <= rtol * abs(want) and err <= atol
        rec = {"mode": mode, "groups": 2, "shards": shards, "weights": [0.0, 1.0], "lnL": lnl, "want": want,
               "site_err": err, "site_atol": atol, "ok": bool(ok)}
        oks = [None] * world
        dist.all_gather_object(oks, rec["ok"])
        rec["ok_all_ranks"] = all(oks)
        out.append(rec)
    return out


def main():
    import torch
    import torch.distributed as dist
    from hyphy_b200 import LikelihoodFunction, Partition, engine
    from hyphy_b200.sharding import shard_bounds, exchange_unique_id, class_groups
    from tests import golden_cases as gc

    name = sys.argv[1]
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("gloo")
    if name == ZERO_WEIGHT_CASE:
        out = {"case": name, "world": world, "layouts": zero_weight_class_groups(world, rank, local, dist)}
        if rank == 0:
            print("MULTIGPU " + json.dumps(out), flush=True)
        dist.barrier()
        dist.destroy_process_group()
        sys.exit(0 if all(r["ok_all_ranks"] for r in out["layouts"]) else 1)
    w, g = gc.load(name)
    pat_golden = np.empty(w.S)
    pat_golden[w.site_to_pattern] = g["site_lnL"]
    out = {"case": name, "world": world, "layouts": []}
    G_max = class_groups(world, w.C)
    for flags, rtol, atol, mode in ((engine.FLAG_FORCE_FP64, 1e-10, 1e-8, "fp64"), (engine.FLAG_DEFAULT, 1e-7, 1e-5, "tc")):
        if mode == "tc" and w.D <= 32:
            continue
        for G in sorted({1, G_max}):
            shards = world // G
            lo, hi = shard_bounds(w.S, shards, rank // G)
            lf = LikelihoodFunction(w, device=local, flags=flags, pattern_slice=slice(lo, hi))
            lf.part.comm_init(world, rank, exchange_unique_id(dist, rank, Partition.comm_unique_id))
            if G > 1:
                lf.part.comm_class_groups(G)
            lf.set_template()
            lf.set_all_compiled()
            lnl, sl, ss = lf.compute(want_sites=True)
            # gathered per-pattern outputs (SURVEY 8e): every rank ends up with the whole alignment's values, in pattern order
            all_l, all_s = lf.part.comm_gather_sites(sl, ss, w.S)
            gather_err = float(np.abs(np.log(all_l) - 64.0 * np.log(2.0) * all_s - pat_golden).max()) if len(all_l) == w.S else float("inf")
            # a second evaluation after a partial update (one leaf's matrices changed and changed back)
            Qt = w.Qt()
            for c in range(w.C):
                lf.part.set_matrices(c, [0], Qt[c, 0][None] * 2.0)
            other = lf.compute(update_nodes=[0])
            for c in range(w.C):
                lf.part.set_matrices(c, [0], Qt[c, 0][None])
            again = lf.compute(update_nodes=[0])
            lf.close()
            site = np.log(sl) - 64.0 * np.log(2.0) * ss
            err = float(np.abs(site - pat_golden[lo:hi]).max())
            rec = {"mode": mode, "groups": G, "shards": shards, "lnL": lnl, "golden": g["lnL"], "rel": abs(lnl - g["lnL"]) / abs(g["lnL"]),
                   "site_err": err, "gathered_site_err": gather_err, "again_equal": again == lnl, "other_differs": other != lnl}
            # every rank must hold the same complete lnL
            box = [None] * world
            dist.all_gather_object(box, lnl)
            rec["identical_on_all_ranks"] = all(b == box[0] for b in box)
            ok = rec["rel"] <= rtol and err <= atol and gather_err <= atol and rec["again_equal"] and rec["other_differs"] and rec["identical_on_all_ranks"]
            rec["ok"] = bool(ok)
            oks = [None] * world
            dist.all_gather_object(oks, rec["ok"])
            rec["ok_all_ranks"] = all(oks)
            out["layouts"].append(rec)
    if rank == 0:
        print("MULTIGPU " + json.dumps(out), flush=True)
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(0 if all(r["ok_all_ranks"] for r in out["layouts"]) else 1)


if __name__ == "__main__":
    main()
