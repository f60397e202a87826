"""Regenerates tests/golden/*.npz by running the UNMODIFIED reference binary (oracle/_ref/hyphy, built from the
reference sources by oracle/Makefile.ref) on seeded synthetic workloads (hyphy_b200/synth.py).

Each fixture holds the reference's lnL and per-site log-likelihoods (ConstructCategoryMatrix SITE_LOG_LIKELIHOODS,
alignment order) plus a checksum of the generated leaf states, so tests can prove they regenerated the same input.
`--runs` writes tests/golden/reference_runs.json instead: what tests/test_host_binding.py compares the patched host
with (the final lnL of an evaluation stream, joint ML ancestral sequences).
Run where the reference binary was built:  python tools/make_golden.py [--runs | name ...]
"""
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from hyphy_b200 import synth            # noqa: E402
from oracle import ref_harness as rh    # noqa: E402

STREAM_CASE, STREAM_EVALS, STREAM_WARM = "mg94_30x100_c4_ambig", 5, 1
ANCESTOR_CASES = ["mg94_8x60_c1", "mg94_8x60_c4_ambig", "c1_hky85_8x500", "mg94_30x100_c4_ambig"]

# name -> constructor.  tests/golden_cases.py imports this table so both sides build identical inputs.
CASES = {
    "c1_hky85_8x500":        lambda: synth.nucleotide_workload(8, 500, ambig_frac=0.01),
    "nuc_300x200_scaling":   lambda: synth.nucleotide_workload(300, 200, mean_t=0.08),
    "mg94_8x60_c1":          lambda: synth.codon_workload(8, 60, 1),
    "mg94_8x60_c4_ambig":    lambda: synth.codon_workload(8, 60, 4, ambig_frac=0.02),
    "mg94_30x100_c4_ambig":  lambda: synth.codon_workload(30, 100, 4, ambig_frac=0.01),
    "c2_mg94_50x1000_c1":    lambda: synth.codon_workload(50, 1000, 1),
    "mg94_200x64_c4_scaling": lambda: synth.codon_workload(200, 64, 4),
    "ns_mg94_200x2000_c4":   lambda: synth.codon_workload(200, 2000, 4),
    # BASELINE.json configs[2] (c3, BUSTED shape: K=3 explicit-form mixture on every branch) and configs[4] (c5)
    "bsrel_12x80_k3":        lambda: synth.bsrel_workload(12, 80),
    "c3_bsrel_100x1500_k3":  lambda: synth.bsrel_workload(100, 1500),
    "c5_mg94_500x5000_c4":   lambda: synth.codon_workload(500, 5000, 4),
}


def checksum(w) -> str:
    h = hashlib.sha256()
    h.update(np.ascontiguousarray(w.leaf_states).tobytes())
    h.update(np.ascontiguousarray(w.pattern_freq).tobytes())
    h.update(np.ascontiguousarray(w.tree.flat_parents).tobytes())
    h.update(np.ascontiguousarray(w.tree.t).tobytes())
    return h.hexdigest()


def reference_runs(out):
    s = rh.run_reference(CASES[STREAM_CASE](), n_evals=STREAM_EVALS, n_warm=STREAM_WARM, per_site=False)
    runs = {"evaluation_stream": {"case": STREAM_CASE, "n_evals": STREAM_EVALS, "n_warm": STREAM_WARM, "loop_lnL": s["loop_lnL"]},
            "ancestors": {name: rh.run_reference(CASES[name](), ancestors=True, per_site=False)["ancestors"] for name in ANCESTOR_CASES}}
    with open(os.path.join(out, "reference_runs.json"), "w") as f:
        json.dump(runs, f, indent=1, sort_keys=True)
        f.write("\n")


def main():
    out = os.path.join(ROOT, "tests", "golden")
    os.makedirs(out, exist_ok=True)
    only = sys.argv[1:]
    if only == ["--runs"]:
        reference_runs(out)
        return
    for name, make in CASES.items():
        if only and name not in only:
            continue
        w = make()
        r = rh.run_reference(w)
        assert r["site_lnL"] is not None and len(r["site_lnL"]) == len(w.site_to_pattern)
        np.savez_compressed(os.path.join(out, name + ".npz"), lnL=np.float64(r["lnL"]), site_lnL=r["site_lnL"],
                            checksum=np.array(checksum(w)), S=np.int64(w.S), sites=np.int64(len(w.site_to_pattern)))
        print(f"{name}: S={w.S} lnL={r['lnL']!r} wall={r['wall']:.1f}s", flush=True)


if __name__ == "__main__":
    main()
