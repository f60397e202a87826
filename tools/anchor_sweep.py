"""Sweep of the anchor threshold of the tensor-core pruning kernel (HB2_ANCHOR_THR): pruning time against lnL error on the
north-star workload and on the deep-tree fixtures.  One process per setting (the threshold is read once per process)."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CODE = r'''
import json, os, sys
sys.path.insert(0, %r)
import numpy as np
from hyphy_b200 import LikelihoodFunction
from tests import golden_cases as gc
out = {"thr": os.environ.get("HB2_ANCHOR_THR")}
for name in ("ns_mg94_200x2000_c4", "mg94_200x64_c4_scaling", "c2_mg94_50x1000_c1"):
    w, g = gc.load(name)
    lf = LikelihoodFunction(w)
    lf.set_template(); lf.set_all_compiled()
    lnl, sl, ss = lf.compute(want_sites=True)
    site = np.log(sl) - 64 * np.log(2.0) * ss
    rec = {"rel": (lnl - g["lnL"]) / abs(g["lnL"]), "site": float(np.abs(site[w.site_to_pattern] - g["site_lnL"]).max())}
    if name.startswith("ns_"):
        lf.part.time_resident(w.class_weights, w.pi, iters=3)
        ms, st, _ = lf.part.time_resident(w.class_weights, w.pi, iters=20)
        rec["pruning_ms"] = float(st[1]); rec["ms"] = ms
    lf.close()
    out[name] = rec
print(json.dumps(out))
''' % ROOT
for thr in ("0.015625", "0.03125", "0.0625", "0.125", "0.25", "2.0"):
    env = dict(os.environ, HB2_ANCHOR_THR=thr)
    r = subprocess.run([sys.executable, "-c", CODE], env=env, capture_output=True, text=True)
    print(r.stdout.strip() or r.stderr[-400:], flush=True)
