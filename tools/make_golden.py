"""Regenerates tests/golden/*.npz by running the UNMODIFIED reference binary (oracle/_ref/hyphy, built from the
reference sources by oracle/Makefile.ref) on seeded synthetic workloads (hyphy_b200/synth.py).

Each fixture holds the reference's lnL and per-site log-likelihoods (ConstructCategoryMatrix SITE_LOG_LIKELIHOODS,
alignment order) plus a checksum of the generated leaf states, so tests can prove they regenerated the same input.
`--runs` writes tests/golden/reference_runs.json instead: what tests/test_host_binding.py compares the patched host
with (the final lnL of an evaluation stream, joint ML ancestral sequences).
`--pinned` writes tests/golden/bsrel_12x80_k3_pinned.npz: MEME's branch-level empirical Bayes procedure
(meme.compute_branch_EBF, MEME.bf:886-944) on every site at once -- see pinned_fixture.
`--impute` writes tests/golden/<case>_impute.npz for IMPUTE_CASES: leaf state imputation
(ReconstructAncestors(MARGINAL, DOLEAVES), MEME's and PRIME's --impute-states) on every site -- see impute_fixture.
`--joint` writes tests/golden/<case>_joint.npz for JOINT_CASES: the joint maximum-likelihood ancestral states
(ReconstructAncestors, as FEL, MEME and PRIME run it per site through ancestral.build) on every site -- see joint_fixture.
Run where the reference binary was built:  python tools/make_golden.py [--runs | --pinned | --impute | --joint | name ...]
"""
import hashlib
import json
import os
import re
import subprocess
import sys
import tempfile

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


PINNED_CASE = "bsrel_12x80_k3"


def pinned_script(w, path_bf, path_fas):
    """The BS-REL script of ref_harness.write_hbl with branch-local mixture weights (as MEME's mixture_aux_weight
    parameters are local to each tested branch), followed by, for every branch b and component k: b's weights set to
    one-hot on k, the per-site log-likelihoods (ConstructCategoryMatrix SITE_LOG_LIKELIHOODS) printed as `PIN b k site
    value`, b's weights restored.  A site's value in the whole-alignment function equals its one-site function's."""
    rh.write_hbl(w, path_bf, path_fas)
    wts = w.meta["mixture"]["weights"]
    K, tree = len(wts), w.tree
    lines = open(path_bf).read().splitlines()
    glob = [i for i, line in enumerate(lines) if re.match(r"global bw\d+ = ", line)]
    assert len(glob) == K
    lines = [line for i, line in enumerate(lines) if i not in glob]         # bw_k: a model parameter local to each branch
    at = max(i for i, line in enumerate(lines) if line.startswith("T.") and ".t := " in line) + 1
    local = [f"T.{tree.names[b]}.bw{k + 1} = {rh._fmt(wts[k])};" for b in range(tree.n_branches) for k in range(K)]
    lines[at:at] = local
    for b in range(tree.n_branches):
        nm = tree.names[b]
        for k in range(K):
            lines += [f"T.{nm}.bw{j + 1} = {1 if j == k else 0};" for j in range(K)]
            lines.append("ConstructCategoryMatrix (sl, lf, SITE_LOG_LIKELIHOODS);")
            lines.append(f'for (k = 0; k < Columns (sl); k += 1) {{ fprintf (stdout, "PIN {b} {k} ", k, " ", Format (sl[k], 30, 16), "\\n"); }}')
        lines += [f"T.{nm}.bw{j + 1} = {rh._fmt(wts[j])};" for j in range(K)]
    with open(path_bf, "w") as f:
        f.write("\n".join(lines) + "\n")


def pinned_fixture(out):
    """tests/golden/bsrel_12x80_k3_pinned.npz: lnL and site_lnL of the branch-local script, and pinned [B*K][sites],
    row b*K + k = every site with branch b (flat id) pinned to component k."""
    w = CASES[PINNED_CASE]()
    K, nb, n = len(w.meta["mixture"]["weights"]), w.tree.n_branches, len(w.site_to_pattern)
    tmp = tempfile.mkdtemp(prefix="hb2ref_")
    bf, fas = os.path.join(tmp, "job.bf"), os.path.join(tmp, "job.fas")
    pinned_script(w, bf, fas)
    proc = subprocess.run([rh.REF_BIN, "CPU=1", bf], cwd=tmp, stdin=subprocess.DEVNULL, capture_output=True, text=True, check=True)
    lnL, site, pinned = None, np.full(n, np.nan), np.full((nb * K, n), np.nan)
    for line in proc.stdout.splitlines():
        f = line.split()
        if line.startswith("LNL="):
            lnL = float(line[4:])
        elif f and f[0] == "SITE":
            site[int(f[1])] = float(f[2])
        elif f and f[0] == "PIN":
            pinned[int(f[1]) * K + int(f[2]), int(f[3])] = float(f[4])
    assert lnL is not None and not np.isnan(site).any() and not np.isnan(pinned).any(), proc.stdout[-2000:]
    np.savez_compressed(os.path.join(out, PINNED_CASE + "_pinned.npz"), lnL=np.float64(lnL), site_lnL=site, pinned=pinned,
                        checksum=np.array(checksum(w)), S=np.int64(w.S), sites=np.int64(n))
    print(f"{PINNED_CASE}_pinned: lnL={lnL!r} rows={nb * K} sites={n}", flush=True)


IMPUTE_CASES = ["bsrel_12x80_k3", "mg94_8x60_c1"]     # mixture layout (K = 3 on every branch), plain layout


def impute_script(w, path_bf, path_fas):
    """The case's script of ref_harness.write_hbl, followed by the marginal reconstruction of the leaves and its support
    matrix: `NAMES` the reconstructed data set's sequence names (the matrix's row order), `DUP` the filter's
    site-to-pattern map, then one `SUP leaf` line per matrix row with its patterns x D entries (pattern-major)."""
    rh.write_hbl(w, path_bf, path_fas, per_site=False)
    lines = ["DataSet anc = ReconstructAncestors (lf, {{0}}, MARGINAL, DOLEAVES);",
             "sm = anc.marginal_support_matrix;",
             "GetString (nms, anc, -1);",
             'for (k = 0; k < Columns (nms); k += 1) { fprintf (stdout, "NAMES ", k, " ", nms[k], "\n"); }',
             "GetDataInfo (dup, flt);",
             'fprintf (stdout, "DUP");',
             'for (k = 0; k < Columns (dup); k += 1) { fprintf (stdout, " ", dup[k]); }',
             'fprintf (stdout, "\n");',
             "for (r = 0; r < Rows (sm); r += 1) {",
             '  fprintf (stdout, "SUP ", r);',
             '  for (c = 0; c < Columns (sm); c += 1) { fprintf (stdout, " ", Format (sm[r][c], 50, 30)); }',
             '  fprintf (stdout, "\n");',
             "}"]
    with open(path_bf, "a") as f:
        f.write("\n".join(lines) + "\n")


def impute_fixture(out, name):
    """tests/golden/<name>_impute.npz: lnL, and support [sites][L][D] -- row l of a site is the reference's support of
    leaf l (flat id, mapped by name) at that site's pattern of the filter (mapped by the filter's site-to-pattern map)."""
    w = CASES[name]()
    L, D, n = w.tree.n_leaves, w.D, len(w.site_to_pattern)
    tmp = tempfile.mkdtemp(prefix="hb2ref_")
    bf, fas = os.path.join(tmp, "job.bf"), os.path.join(tmp, "job.fas")
    impute_script(w, bf, fas)
    proc = subprocess.run([rh.REF_BIN, "CPU=1", bf], cwd=tmp, stdin=subprocess.DEVNULL, capture_output=True, text=True, check=True)
    lnL, names, dup, rows = None, {}, None, {}
    for line in proc.stdout.splitlines():
        f = line.split()
        if line.startswith("LNL="):
            lnL = float(line[4:])
        elif f and f[0] == "NAMES":
            names[int(f[1])] = f[2]
        elif f and f[0] == "DUP":
            dup = np.array([int(x) for x in f[1:]], dtype=np.int64)
        elif f and f[0] == "SUP":
            rows[int(f[1])] = np.array([float(x) for x in f[2:]])
    assert lnL is not None and dup is not None and len(dup) == n and len(rows) == L == len(names), proc.stdout[-2000:]
    n_pat = int(dup.max()) + 1
    leaf_of = {nm: l for l, nm in enumerate(w.tree.names[:L])}
    support = np.full((n, L, D), np.nan)
    for r, row in rows.items():
        assert row.shape == (n_pat * D,)
        support[:, leaf_of[names[r]], :] = row.reshape(n_pat, D)[dup]
    assert not np.isnan(support).any()
    for p in range(w.S):                        # sites of one pattern of the engine's compression share their rows
        sites = np.nonzero(w.site_to_pattern == p)[0]
        assert np.all(support[sites] == support[sites[:1]]), p
    np.savez_compressed(os.path.join(out, name + "_impute.npz"), lnL=np.float64(lnL), support=support,
                        checksum=np.array(checksum(w)), S=np.int64(w.S), sites=np.int64(n))
    print(f"{name}_impute: lnL={lnL!r} leaves={L} sites={n} filter patterns={n_pat}", flush=True)


# mixture layout (K = 3 on every branch), plain layout, and a gap-rich plain case ('---', N and R/Y codons, unresolved
# cherries) that nothing but its fixture builds or loads
JOINT_CASES = {"bsrel_12x80_k3": CASES["bsrel_12x80_k3"], "mg94_8x60_c1": CASES["mg94_8x60_c1"],
               "mg94_8x60_c1_gaps": lambda: synth.codon_workload(8, 60, 1, ambig_frac=0.5)}


def joint_script(w, path_bf, path_fas):
    """The case's script of ref_harness.write_hbl, followed by the joint reconstruction: `NAMES` the reconstructed data
    set's sequence names, `DUP` the filter's site-to-pattern map, then one `ANC k sequence` line per internal node."""
    rh.write_hbl(w, path_bf, path_fas, per_site=False)
    lines = ["DataSet anc = ReconstructAncestors (lf);",
             "GetString (nms, anc, -1);",
             'for (k = 0; k < Columns (nms); k += 1) { fprintf (stdout, "NAMES ", k, " ", nms[k], "\n"); }',
             "GetDataInfo (dup, flt);",
             'fprintf (stdout, "DUP");',
             'for (k = 0; k < Columns (dup); k += 1) { fprintf (stdout, " ", dup[k]); }',
             'fprintf (stdout, "\n");',
             "DataSetFilter ancf = CreateFilter (anc, 1);",
             'for (k = 0; k < ancf.species; k += 1) { GetDataInfo (aSeq, ancf, k); fprintf (stdout, "ANC ", k, " ", aSeq, "\n"); }']
    with open(path_bf, "a") as f:
        f.write("\n".join(lines) + "\n")


def joint_fixture(out, name):
    """tests/golden/<name>_joint.npz: states [sites][I] -- entry i of a site is the reference's joint ML state of internal
    node i (mapped by name) as a sense-codon index of synth's codon table, -1 for '---' -- and the workload checksum."""
    w = JOINT_CASES[name]()
    L, I, n = w.tree.n_leaves, w.tree.n_internal, len(w.site_to_pattern)
    tmp = tempfile.mkdtemp(prefix="hb2ref_")
    bf, fas = os.path.join(tmp, "job.bf"), os.path.join(tmp, "job.fas")
    joint_script(w, bf, fas)
    proc = subprocess.run([rh.REF_BIN, "CPU=1", bf], cwd=tmp, stdin=subprocess.DEVNULL, capture_output=True, text=True, check=True)
    names, dup, seqs = {}, None, {}
    for line in proc.stdout.splitlines():
        f = line.split()
        if f and f[0] == "NAMES":
            names[int(f[1])] = f[2]
        elif f and f[0] == "DUP":
            dup = np.array([int(x) for x in f[1:]], dtype=np.int64)
        elif f and f[0] == "ANC":
            seqs[int(f[1])] = f[2]
    assert dup is not None and len(dup) == n and len(seqs) == I == len(names), proc.stdout[-2000:]
    node_of = {nm: i for i, nm in enumerate(w.tree.names[L:L + I - 1])}
    unnamed = [nm for nm in names.values() if nm not in node_of]
    assert len(unnamed) == 1, unnamed           # the newick leaves the root unnamed: the binary names it itself
    node_of[unnamed[0]] = I - 1
    code = {synth.codon_str(c): k for k, c in enumerate(synth.SENSE)}
    code["---"] = -1
    states = np.full((n, I), -2, dtype=np.int64)
    for k, seq in seqs.items():
        assert len(seq) == 3 * n, (k, len(seq))
        states[:, node_of[names[k]]] = [code[seq[3 * j:3 * j + 3]] for j in range(n)]
    assert np.all(states >= -1)
    for p in range(w.S):                        # sites of one pattern of the engine's compression share their states
        sites = np.nonzero(w.site_to_pattern == p)[0]
        assert np.all(states[sites] == states[sites[:1]]), p
    np.savez_compressed(os.path.join(out, name + "_joint.npz"), states=states, checksum=np.array(checksum(w)),
                        S=np.int64(w.S), sites=np.int64(n))
    print(f"{name}_joint: internal nodes={I} sites={n} unresolved={int((states < 0).sum())}", flush=True)


def main():
    out = os.path.join(ROOT, "tests", "golden")
    os.makedirs(out, exist_ok=True)
    only = sys.argv[1:]
    if only == ["--runs"]:
        reference_runs(out)
        return
    if only == ["--pinned"]:
        pinned_fixture(out)
        return
    if only == ["--joint"]:
        for name in JOINT_CASES:
            joint_fixture(out, name)
        return
    if only == ["--impute"]:
        for name in IMPUTE_CASES:
            impute_fixture(out, name)
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
