#!/usr/bin/env python
"""Runs the reference's OWN regression batch files (tests/hbltests, copied to oracle/_ref/host/hbltests by apply_hooks.py) through
a HyPhy binary and extracts what they report: every `Log Likelihood = x` a fitted likelihood function prints, and the
test's PASSED / FAILED verdict.

    python host/regress.py expect   # where the reference sources were built: run the UNMODIFIED reference binary
                                    # (oracle/_ref/hyphy) and write tests/golden/hbltests_expected.json
    python host/regress.py check    # on the GPU: run the PATCHED binary (oracle/_ref/host/hyphy, engine on, its default fp64
                                    # kernels) and compare;  `tc` = the same with HYPHY_B200_TC=1, `cpu` = engine off

TEST INFRASTRUCTURE (it drives the unmodified reference as the checker); the product is the patched binary it checks.
"""
from __future__ import annotations

import json
import os
import re
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "oracle", "_ref", "host")
REF_BIN = os.path.join(ROOT, "oracle", "_ref", "hyphy")
HOST_BIN = os.path.join(BUILD, "hyphy")
EXPECTED = os.path.join(ROOT, "tests", "golden", "hbltests_expected.json")

# reference batch files that exercise the likelihood hot path through different host modes (relative to tests/hbltests)
TESTS = [
    "SimpleOptimizations/SmallCodon.bf",            # golden lnL -3189.516375 (SmallCodon.bf:37)
    "SimpleOptimizations/SmallCodonLocal.bf",       # branch-local parameters -> single-branch updates
    "SimpleOptimizations/IntermediateProtein.bf",   # 20 states
    "SimpleOptimizations/LargeNuc.bf",
    "SimpleOptimizations/multi-part-codon.bf",      # several partitions in one likelihood function
    "SimpleOptimizations/TwoSequenceTest.bf",       # two-sequence special case (likefunc.cpp:11260): stays on the host's own path
    "REL/GTR_G_I.bf",                               # category variables: per-class ComputeBlock + host combination
    "REL/NY.bf",
    "REL/ModelMixture.bf",
    "HMM/SmallNuc.bf",                              # HMM category variables
    "HMM/RateHMM.bf",
    "Ancestors/NucRVAncestors.bf",                  # ancestral reconstruction with rate variation
    "SpecializedOptimizations/SiteLikelihood.bf",   # per-site likelihoods (SURVEY §4)
    "SpecializedOptimizations/MEME.bf",
    "Trickier/NonReversibleWithDynamicFrequencies.bf",  # non-reversible NRM model, frequencies not at equilibrium
    # the five analyses north_star names, as the reference's own workflow tests drive them (libv3, CD2.nex)
    "libv3/FEL.wbf",
    "libv3/BUSTED.wbf",
    "libv3/MEME.wbf",
    "libv3/ABSREL.wbf",
    "libv3/RELAX.wbf",
]
# (other batch files under tests/hbltests are broken at this reference commit with the unmodified binary itself --
#  syntax errors, missing template files -- and carry no information about the binding)

# RELAX's later fits land in different local optima from run to run with the UNMODIFIED binary already (thread count
# changes the summation order and with it the optimiser's path): only its first three fits are compared
STABLE_PREFIX = {"libv3/RELAX.wbf": 3}

# batch files that read their data by a path relative to the working directory rather than to themselves: they run in
# their own directory (of the private copy)
RUN_IN_OWN_DIR = {"Trickier/NonReversibleWithDynamicFrequencies.bf"}
# batch files that print no log-likelihood: a wrapper executes the file unchanged with soft assertions (a failed one ends
# the file, not the run), then prints this expression of its results.  The unmodified binary itself misses this file's own
# expected value by 0.018 (tolerance 0.01), so its verdict alone says little.
PRINT_AFTER = {"Trickier/NonReversibleWithDynamicFrequencies.bf": "res[1][0]"}

_WORK = None


def work_tree():
    """A private, writable copy of the batch-file library and the regression tests: the batch files write their result
    files (JSON reports, optimisation logs) next to themselves, and the build tree may be read-only for whoever runs them."""
    global _WORK
    if _WORK is None:
        _WORK = tempfile.mkdtemp(prefix="hb2lib_")
        for sub in ("res", "hbltests"):
            shutil.copytree(os.path.join(BUILD, sub), os.path.join(_WORK, sub), copy_function=shutil.copyfile)
        for d, _, files in os.walk(_WORK):           # copytree keeps the directories' modes: make them writable
            os.chmod(d, 0o755)
            for f in files:
                os.chmod(os.path.join(d, f), 0o644)
    return _WORK


LL = re.compile(r"(?:Log Likelihood|Log\(L\))\s*=\s*(-?[0-9]+\.?[0-9]*(?:[eE][-+]?[0-9]+)?)")


def run(binary, test, env_extra=None, timeout=900, threads=0):
    work = work_tree()
    path = os.path.join(work, "hbltests", test)
    env = dict(os.environ)
    env.update(env_extra or {})
    tmp = tempfile.mkdtemp(prefix="hb2reg_")
    cwd = os.path.dirname(path) if test in RUN_IN_OWN_DIR else tmp
    if test in PRINT_AFTER:
        wrapper = os.path.join(tmp, "wrapper.bf")
        with open(wrapper, "w") as f:
            f.write(f'ASSERTION_BEHAVIOR = 1;\nExecuteAFile ("{path}");\nfprintf (stdout, "\\nLog Likelihood = ", {PRINT_AFTER[test]}, "\\n");\n')
        path = wrapper
    t0 = time.time()
    args = [binary, f"LIBPATH={os.path.join(work, 'res')}"] + ([f"CPU={threads}"] if threads else []) + [path]
    try:
        pr = subprocess.run(args, cwd=cwd, stdin=subprocess.DEVNULL, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                            text=True, env=env, timeout=timeout)
        out, rc = pr.stdout, pr.returncode
    except subprocess.TimeoutExpired as e:
        out, rc = (e.stdout or b"").decode("utf-8", "replace") if isinstance(e.stdout, bytes) else (e.stdout or ""), -9
    verdict = "passed" if "[TEST PASSED]" in out else "failed" if "[TEST FAILED]" in out else "error" if rc != 0 else "none"
    if os.environ.get("HB2_REGRESS_KEEP"):          # debugging aid: full transcript next to the other gpurun outputs
        os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
        tag = "tc" if (env_extra or {}).get("HYPHY_B200_TC") else "cpu" if (env_extra or {}).get("HYPHY_B200") == "0" else "fp64"
        with open(os.path.join(ROOT, "gpurun_out", "regress_" + test.replace("/", "_") + "." + tag + ".txt"), "w") as f:
            f.write(out)
    return {"lnL": [float(x) for x in LL.findall(out)], "verdict": verdict, "rc": rc, "seconds": round(time.time() - t0, 2),
            "engine": [l for l in out.splitlines() if l.startswith("[hyphy_b200]")][-4:], "tail": out[-600:] if verdict in ("error",) else ""}


def main():
    mode = sys.argv[1] if len(sys.argv) > 1 else "check"
    only = sys.argv[2:]
    tests = [t for t in TESTS if not only or t in only]
    if mode == "expect":
        exp = json.load(open(EXPECTED)) if (os.path.exists(EXPECTED) and only) else {}
        for t in tests:
            r = run(REF_BIN, t, threads=4)
            exp[t] = {"lnL": r["lnL"], "verdict": r["verdict"], "rc": r["rc"], "seconds_cpu": r["seconds"]}
            print(t, exp[t], flush=True)
        json.dump(exp, open(EXPECTED, "w"), indent=1, sort_keys=True)
        return 0
    exp = json.load(open(EXPECTED))
    bad = 0
    for t in tests:
        if t not in exp:
            continue
        extra = {"HYPHY_B200_VERBOSE": "1"}
        if mode == "cpu":
            extra["HYPHY_B200"] = "0"
        if mode == "tc":
            extra["HYPHY_B200_TC"] = "1"
        r = run(HOST_BIN, t, extra)
        e = exp[t]
        # fitted log-likelihoods: optimiser end points, printed with 2 decimals by the workflows -> 0.05 absolute
        n = STABLE_PREFIX.get(t, len(e["lnL"]))
        ok = r["verdict"] == e["verdict"] and r["rc"] == e.get("rc", 0) and (t in STABLE_PREFIX or len(r["lnL"]) == len(e["lnL"])) and all(
            abs(a - b) <= 0.05 + 1e-6 * abs(b) for a, b in zip(r["lnL"][:n], e["lnL"][:n]))
        bad += not ok
        print(json.dumps({"test": t, "ok": ok, "got": r, "expected": e}), flush=True)
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
