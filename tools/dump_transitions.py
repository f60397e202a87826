"""Every transition matrix of the north-star workload of bench.py (200 taxa x 2000 codons, MG94xREV, 4 omega classes), as
the engine holds it after a hand-over: hb2_read_transition for every (class, branch) slot, after a compiled hand-over
and after a dense one.  Writes OUT/transitions_compiled.npy and OUT/transitions_dense.npy ([C][B][D][D] float64) and
prints their sha256, so that two builds can be compared byte for byte."""
import argparse
import hashlib
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, metavar="DIR", help="output directory")
    args = ap.parse_args()
    from hyphy_b200 import synth, LikelihoodFunction
    import bench

    os.makedirs(args.out, exist_ok=True)
    w = synth.codon_workload(bench.WORKLOAD["taxa"], bench.WORKLOAD["codons"], bench.WORKLOAD["classes"])
    lf = LikelihoodFunction(w, device=0)
    lf.set_template()
    for route in ("compiled", "dense"):
        if route == "compiled":
            lf.set_all_compiled()
        else:
            lf.set_all_matrices()
        lnl = lf.compute()
        P = np.stack([np.stack([lf.part.read_transition(c, b) for b in range(w.tree.n_branches)]) for c in range(w.C)])
        np.save(os.path.join(args.out, f"transitions_{route}.npy"), P)
        print(f"{route}: lnL={lnl!r} sha256={hashlib.sha256(P.tobytes()).hexdigest()} shape={P.shape}")
    lf.close()


if __name__ == "__main__":
    main()
