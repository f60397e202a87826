"""Evaluation stream of the north-star workload through the PATCHED HyPhy binary (oracle/_ref/host/hyphy): evaluations/s of HBL
`LFCompute` for both hand-over routes (compiled formula values / dense Q*t) and both precisions, next to the engine's own
account of where the time went (HYPHY_B200_VERBOSE)."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from hyphy_b200 import synth          # noqa: E402
from oracle import ref_harness as rh  # noqa: E402

HOST = os.path.join(ROOT, "oracle", "_ref", "host", "hyphy")
n = int(sys.argv[1]) if len(sys.argv) > 1 else 20
w = synth.codon_workload(200, 2000, 4)
out = []
for name, env in (("compiled,tc", {"HYPHY_B200_TC": "1"}), ("dense,tc", {"HYPHY_B200_TC": "1", "HYPHY_B200_DENSE": "1"}),
                  ("compiled,fp64", {}), ("dense,fp64", {"HYPHY_B200_DENSE": "1"}), ("cpu (engine off, 1 thread)", {"HYPHY_B200": "0"})):
    e = dict(env, HYPHY_B200_VERBOSE="1")
    r = rh.run_reference(w, n_evals=n if "cpu" not in name else 3, n_warm=2, per_site=False, binary=HOST, env_extra=e)
    k = n if "cpu" not in name else 3
    rec = {"route": name, "evals_per_s": k / r["loop_seconds"], "lnL": r["lnL"], "engine": r["engine"][-1:] }
    out.append(rec)
    print(json.dumps(rec), flush=True)
