"""TEST / BASELINE INFRASTRUCTURE -- not part of the product path.

Drives the UNMODIFIED reference binary (oracle/_ref/hyphy, built by oracle/Makefile.ref straight from the
reference sources) on a synthetic workload: writes a FASTA + a self-contained HBL script (no libv3, no
LIBPATH needed, so it also runs on the GPU box where /root/reference does not exist), runs it, and parses
lnL, per-site log-likelihoods and wall time.

What the generated HBL exercises in the reference: `LFCompute` (batchlanruntime.cpp:2205) ->
`_LikelihoodFunction::Compute` (likefunc.cpp:2421) -> `ComputeBlock` (likefunc.cpp:10783) ->
`ExponentiateMatrices` + `ComputeTreeBlockByBranch`; with a category variable the path goes through
`PopulateConditionalProbabilities` (likefunc2.cpp:484).  Model syntax follows the reference's own tests
(tests/hbltests/SimpleOptimizations/SmallCodon.bf:56-661, res/TemplateBatchFiles/2RatesAnalyses/PARRIS_M3.def:21-23).

Only tests/, bench.py (cpu_baseline / --impl reference) and tools/make_golden.py import this module.
"""
from __future__ import annotations

import os
import re
import subprocess
import tempfile
import time

import numpy as np

from hyphy_b200 import synth

HERE = os.path.dirname(os.path.abspath(__file__))
REF_BIN = os.path.join(HERE, "_ref", "hyphy")


def have_reference() -> bool:
    return os.path.isfile(REF_BIN) and os.access(REF_BIN, os.X_OK)


def _fmt(x: float) -> str:
    return repr(float(x))


def write_hbl(w: synth.Workload, path_bf: str, path_fas: str, n_evals: int = 0, threads: int = 0,
              per_site: bool = True, n_warm: int = 0, ancestors: bool = False) -> None:
    """Emit FASTA + HBL for workload `w`.  n_evals>0 appends the timed full-evaluation loop (one global
    parameter perturbed by 1e-4 relative each time, SURVEY §8d); threads>0 enables OpenMP inside LFCompute
    the only way the unmodified reference allows (NUMBER_THREADS + an Optimize call, likefunc.cpp:223-227)."""
    assert w.site_chars is not None, "workload has no character data for the reference"
    tree = w.tree
    with open(path_fas, "w") as f:
        for k in range(tree.n_leaves):
            f.write(f">{tree.names[k]}\n{w.site_chars[k]}\n")
    kind = w.meta["kind"]
    o = []
    o.append(f'DataSet ds = ReadDataFile ("{path_fas}");')
    if kind == "codon":
        o.append('DataSetFilter flt = CreateFilter (ds,3,"","","TAA,TAG,TGA");')
        th = dict(zip(["AC", "AG", "AT", "CG", "CT", "GT"], w.meta["theta"]))
        for nm in ["AC", "AT", "CG", "CT", "GT"]:
            o.append(f"global {nm} = {_fmt(th[nm])};")
        mix = w.meta.get("mixture")
        omegas = w.meta["omegas"]
        if mix:
            # explicit-form model: P_b = sum_k bw_k * Exp(Q_k), Q_k = MG94 with omega_k (BranchSiteREL.bf:272-277 builds its
            # models the same way); rates carry the frequencies, the diagonal is filled by the evaluator (matrix.cpp:3296)
            K = len(mix["omegas"])
            for k in range(K):
                o.append(f"global omega{k + 1} = {_fmt(mix['omegas'][k])};")
                o.append(f"global bw{k + 1} = {_fmt(mix['weights'][k])};")
            entries = synth.mg94_entries(w.meta["theta"], np.array(w.meta["posfreq"]))
            for k in range(K):
                o.append(f"Q{k + 1} = {{61,61}};")
                for i, j, pf, nonsyn, nm in entries:
                    terms = ["t"]
                    if nm != "AG":
                        terms.append(nm)
                    if nonsyn:
                        terms.append(f"omega{k + 1}")
                    terms.append(_fmt(pf))
                    o.append(f"Q{k + 1}[{i}][{j}] := {'*'.join(terms)};")
            o.append("freqs = {61,1};")
            for k, p in enumerate(w.pi):
                o.append(f"freqs[{k}][0] = {_fmt(p)};")
            expr = "+".join(f"Exp(Q{k + 1})*bw{k + 1}" for k in range(K))
            o.append(f'Model M = ("{expr}", freqs, EXPLICIT_FORM_MATRIX_EXPONENTIAL);')
        else:
          if len(omegas) == 1:
            o.append(f"global omega = {_fmt(omegas[0])};")
          else:
            wts = ",".join(_fmt(x) for x in w.class_weights)
            rts = ",".join(_fmt(x) for x in omegas)
            o.append(f"catW = {{{{{wts}}}}};")
            o.append(f"catR = {{{{{rts}}}}};")
            o.append(f"category omega = ({len(omegas)}, catW, MEAN, , catR, 0, 1e25);")
          o.append("Q = {61,61};")
          assert abs(th["AG"] - 1.0) < 1e-15
          for i, j, pf, nonsyn, nm in synth.mg94_entries(w.meta["theta"], np.array(w.meta["posfreq"])):
            terms = ["t"]
            if nm != "AG":
                terms.append(nm)
            if nonsyn:
                terms.append("omega")
            terms.append(_fmt(pf))
            o.append(f"Q[{i}][{j}] := {'*'.join(terms)};")
          o.append("freqs = {61,1};")
          for k, p in enumerate(w.pi):
            o.append(f"freqs[{k}][0] = {_fmt(p)};")
          o.append("Model M = (Q, freqs, 0);")
        perturb_name, perturb_base = "AC", th["AC"]
    elif kind == "nuc":
        o.append("DataSetFilter flt = CreateFilter (ds,1);")
        o.append(f"global kappa = {_fmt(w.meta['kappa'])};")
        o.append("Q = {{*,t,kappa*t,t}{t,*,t,kappa*t}{kappa*t,t,*,t}{t,kappa*t,t,*}};")
        fr = ",".join("{" + _fmt(p) + "}" for p in w.meta["freqs"])
        o.append(f"freqs = {{{fr}}};")
        o.append("Model M = (Q, freqs, 1);")
        perturb_name, perturb_base = "kappa", w.meta["kappa"]
    else:
        raise ValueError(kind)
    o.append(f"Tree T = {tree.newick};")
    for b in range(tree.n_branches):
        # branch parameters are constants (:=) so a truncated Optimize only sees the globals
        o.append(f"T.{tree.names[b]}.t := {_fmt(tree.t[b])};")
    o.append("LikelihoodFunction lf = (flt, T);")
    if threads > 0:
        o.append(f"NUMBER_THREADS = {threads};")
        o.append("OPTIMIZATION_TIME_HARD_LIMIT = 1; MAXIMUM_OPTIMIZATION_ITERATIONS = 1; VERBOSITY_LEVEL = -1;")
        o.append("Optimize (res_trunc, lf);")
        if kind == "codon":
            for nm in ["AC", "AT", "CG", "CT", "GT"]:
                o.append(f"{nm} = {_fmt(th[nm])};")
            if len(w.meta["omegas"]) == 1 and not w.meta.get("mixture"):
                o.append(f"omega = {_fmt(w.meta['omegas'][0])};")
        else:
            o.append(f"kappa = {_fmt(w.meta['kappa'])};")
    o.append("LFCompute (lf, LF_START_COMPUTE);")
    o.append("LFCompute (lf, l0);")
    o.append('fprintf (stdout, "LNL=", Format (l0, 30, 16), "\\n");')
    if n_evals > 0:
        if n_warm > 0:
            o.append(f"for (k = 0; k < {n_warm}; k += 1) {{ {perturb_name} = {_fmt(perturb_base)} * (1 - 0.0001*(k+1)); LFCompute (lf, l1); }}")
        o.append('fprintf (stdout, "LOOP_BEGIN\\n");')
        o.append(f"for (k = 0; k < {n_evals}; k += 1) {{ {perturb_name} = {_fmt(perturb_base)} * (1 + 0.0001*(k+1)); LFCompute (lf, l1); }}")
        o.append('fprintf (stdout, "LOOP_END ", Format (l1, 30, 16), "\\n");')
        o.append(f"{perturb_name} = {_fmt(perturb_base)};")
    o.append("LFCompute (lf, LF_DONE_COMPUTE);")
    if per_site:
        o.append("ConstructCategoryMatrix (sl, lf, SITE_LOG_LIKELIHOODS);")
        o.append('for (k = 0; k < Columns (sl); k += 1) { fprintf (stdout, "SITE ", k, " ", Format (sl[k], 30, 16), "\\n"); }')
    if ancestors:
        # joint ML ancestral reconstruction (likefunc2.cpp:308 -> tree.cpp:4209), printed the way the reference's own
        # Ancestors/NucAncestors.bf reads it back
        o.append("DataSet anc = ReconstructAncestors (lf);")
        o.append("DataSetFilter ancf = CreateFilter (anc,1);")
        o.append('for (k = 0; k < ancf.species; k += 1) { GetDataInfo (aSeq, ancf, k); fprintf (stdout, "ANC ", k, " ", aSeq, "\\n"); }')
    with open(path_bf, "w") as f:
        f.write("\n".join(o) + "\n")


def run_reference(w: synth.Workload, n_evals: int = 0, threads: int = 0, per_site: bool = True,
                  timeout: float = 3600.0, workdir: str | None = None, n_warm: int = 0, binary: str | None = None,
                  env_extra: dict | None = None, ancestors: bool = False) -> dict:
    """Run the reference binary on `w`.  Returns {"lnL", "site_lnL" (np array, alignment order) or None,
    "loop_seconds" (wall time between LOOP_BEGIN and LOOP_END, measured on this side of the pipe), "wall"}.
    binary: another HyPhy executable fed the same script -- the PATCHED host (oracle/_ref/host/hyphy) in tests/test_host_binding.py."""
    if binary is None and not have_reference():
        raise RuntimeError(f"reference binary missing: {REF_BIN} (build with make -f oracle/Makefile.ref)")
    tmp = workdir or tempfile.mkdtemp(prefix="hb2ref_")
    bf, fas = os.path.join(tmp, "job.bf"), os.path.join(tmp, "job.fas")
    write_hbl(w, bf, fas, n_evals, threads, per_site, n_warm, ancestors)
    env = dict(os.environ)
    env.update(env_extra or {})
    if threads > 0:
        env["OMP_NUM_THREADS"] = str(threads)
    t0 = time.time()
    proc = subprocess.Popen([binary or REF_BIN, f"CPU={max(threads, 1)}", bf], cwd=tmp, stdin=subprocess.DEVNULL,
                            stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env)
    lnL, sites, t_begin, t_end, loop_lnl, tail, engine_lines = None, {}, None, None, None, [], []
    anc = {}
    try:
        for line in proc.stdout:
            tail.append(line)
            tail = tail[-30:]
            if line.startswith("[hyphy_b200]"):
                engine_lines.append(line.strip())
            if line.startswith("LNL="):
                lnL = float(line[4:])
            elif line.startswith("LOOP_BEGIN"):
                t_begin = time.time()
            elif line.startswith("LOOP_END"):
                t_end = time.time()
                loop_lnl = float(line.split()[1])
            elif line.startswith("SITE "):
                _, k, v = line.split()
                sites[int(k)] = float(v)
            elif line.startswith("ANC "):
                _, k, v = line.split()
                anc[int(k)] = v
            if time.time() - t0 > timeout:
                proc.kill()
                raise TimeoutError("reference run exceeded timeout")
        proc.wait()
    finally:
        if proc.poll() is None:
            proc.kill()
    if lnL is None:
        raise RuntimeError("reference produced no lnL; tail:\n" + "".join(tail))
    site_arr = None
    if sites:
        site_arr = np.array([sites[k] for k in range(len(sites))])
    return {"lnL": lnL, "site_lnL": site_arr, "loop_lnL": loop_lnl, "engine": engine_lines,
            "ancestors": [anc[k] for k in range(len(anc))],
            "loop_seconds": (t_end - t_begin) if (t_begin and t_end) else None, "wall": time.time() - t0}
