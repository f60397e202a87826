#!/usr/bin/env python
"""Builds the PATCHED host: copies the reference's sources into a scratch build tree and inserts the handful of hook calls
that bind libhyphy_b200.so behind `_LikelihoodFunction::ComputeBlock` (SURVEY.md §8b; INTEGRATION.md walks through them).

    python host/apply_hooks.py --ref <HyPhy source tree> [--out oracle/_ref/host]

Every insertion is anchored on a short text fragment of the reference source (so a maintainer can find the place) and
adds only calls into host/hb2_hyphy_hooks.{h,cpp} -- this repository contains the ADDED lines only, never reference
code; the build tree (oracle/_ref/host, git-ignored) is where the two meet.  The script fails loudly when an anchor is
missing or ambiguous, i.e. when the reference has moved on and the binding needs a maintainer's eyes.
"""
from __future__ import annotations

import argparse
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))

INCLUDE = '#include "hb2_hyphy_hooks.h"   // hyphy_b200\n'

# (file, anchor text, where, inserted text, note)   where: "before" | "after" the LINE containing the anchor;
# an integer shifts the insertion point by that many lines (negative = earlier).
HOOKS = [
    # ---- tree.h: the flat parent table is protected; the glue reads it through a friend ------------------------------
    ("core/include/tree.h", "class _TheTree : public _TreeTopology {", "after",
     "  friend struct hb2_hooks_access;   // hyphy_b200: read access to flatParents\n",
     "friend declaration"),
    # ---- matrix.h: the compiled form of a model matrix (cmd, theIndex, lDim) is private -------------------------------
    ("core/include/matrix.h", "class _Matrix : public _MathObject {", "after",
     "  friend struct hb2_hooks_access;   // hyphy_b200: read access to the compiled formula data\n",
     "friend declaration"),
    # ---- likefunc.h: one opaque slot per likelihood function ---------------------------------------------------------
    ("core/include/likefunc.h", "  hyFloat **conditionalInternalNodeLikelihoodCaches, **siteScalingFactors,", ("after", 1),
     "  void *hb2_state = nullptr;   // hyphy_b200: engine partitions, parallel to theTrees\n",
     "state slot next to the host caches (likefunc.h:1291)"),
    # ---- likefunc.cpp ------------------------------------------------------------------------------------------------
    ("core/likefunc.cpp", '#include "likefunc.h"', "after", INCLUDE, "include"),
    ("core/likefunc.cpp", "    OCLEval[i].init(patternCount, theFilter->GetDimension(),", ("before", -1),
     "    if (leafCount > 1UL)   // hyphy_b200: SetupLFCaches, end of the per-partition loop body (likefunc.cpp:4311-4317)\n"
     "      hb2_hooks::create(hb2_state, theTrees.lLength, i, cT, theFilter, conditionalTerminalNodeStateFlag[i], ambigs,\n"
     "                        ambig_resolution_count - 1L);\n",
     "create one engine partition per tree where the OpenCL evaluator used to be initialised"),
    ("core/likefunc.cpp", "        t->ExponentiateMatrices(*matrices, MAX(1, GetThreadCount()), catID);", ("before", -1),
     "      // hyphy_b200: while this scope is alive _CalcNode::SetCompExp hands the queued matrices to the engine\n"
     "      hb2_hooks::Scope hb2_scope(hb2_hooks::partition(hb2_state, index));\n",
     "ComputeBlock: divert the matrix queue (likefunc.cpp:10978)"),
    ("core/likefunc.cpp", "        t->ExponentiateMatrices(*matrices, MAX(1, GetThreadCount()), catID);", ("after", 1),
     "      if (hb2_scope.part())   // hyphy_b200: replaces likefunc.cpp:10984-11259 (branch cache, OpenMP pruning, Neumaier sum, scaler correction)\n"
     "        return hb2_hooks::compute_block(hb2_scope.part(), t, catID, *branches, siteRes, scc, branchIndex, branchValues);\n",
     "ComputeBlock: pruning + root reduction on the engine"),
    ("core/likefunc.cpp", "  delete_array_elements_and_self(conditionalInternalNodeLikelihoodCaches,", "before",
     "  hb2_hooks::destroy_all(hb2_state);   // hyphy_b200: pair of SetupLFCaches\n",
     "DeleteCaches (likefunc.cpp:10594)"),
    # ---- likefunc2.cpp: ancestral reconstruction reads matrices and conditionals on the host -----------------------------
    ("core/likefunc2.cpp", '#include "likefunc.h"', "after", INCLUDE, "include"),
    ("core/likefunc2.cpp", "    _List *expandedMap = dsf->ComputePatternToSiteMap(), *thisSet;", "before",
     "    // hyphy_b200: joint reconstruction / sampling read P and the internal-node conditionals on the host\n"
     "    hb2_hooks::materialize(hb2_hooks::partition(hb2_state, partIndex), tree, dsf, conditionalInternalNodeLikelihoodCaches[partIndex],\n"
     "                           (_SimpleList *)optimalOrders.list_data[partIndex]);\n",
     "ReconstructAncestors (likefunc2.cpp:411): device -> host copies"),
    # ---- tree.cpp: the node-support reader behind ConstructCategoryMatrix (tree) ---------------------------------------------------
    ("core/tree.cpp", '#include "tree.h"', "after", INCLUDE, "include"),
    ("core/tree.cpp", "  IntPopulateLeaves(dsf, site_index);", "before",
     "  if (site_index == 0L) hb2_hooks::materialize_tree(this);   // hyphy_b200: the loop below reads GetCompExp()->theData (tree.cpp:2589)\n",
     "RecoverNodeSupportStates (tree.cpp:2533): device -> host copy of the transition matrices"),
    # ---- calcnode.cpp: SetCompExp is where every matrix of the queue ends up -------------------------------------------
    ("core/calcnode.cpp", '#include "calcnode.h"', "after", INCLUDE, "include"),
    ("core/calcnode.cpp", "void _CalcNode::SetCompExp(_Matrix *m, long catID, bool do_exponentiation) {", "after",
     "  long const hb2_cat = catID;   // hyphy_b200: the rate class as ComputeBlock numbers it (before the category remap)\n",
     "remember the global class index"),
    ("core/calcnode.cpp", "        temp = (_Matrix *)myModelMatrix->MultByFreqs(theModel, true);", ("before", -3),
     "      // hyphy_b200: compiled hand-over -- the formula VALUES go to the engine, which scatters, multiplies by the\n"
     "      // frequencies, fills the diagonal and exponentiates; the if below makes the host's own assembly conditional\n"
     "      _Matrix *hb2_ph = (!isExplicitForm && queue && tags && !storeRateMatrix)\n"
     "                            ? hb2_hooks::compiled(this, myModelMatrix, theModel, categID, GetCompExp(totalCategs > 1 ? categID : -1))\n"
     "                            : nil;\n"
     "      if (!hb2_ph)\n",
     "RecomputeMatrix: skip EvaluateSimple's scatter + MultByFreqs (calcnode.cpp:620-625)"),
    ("core/calcnode.cpp", "      if (storeRateMatrix) {", "before",
     "      if (hb2_ph) {   // hyphy_b200: nothing to queue for ExponentiateMatrices; the node keeps a shape-only matrix\n"
     "        hb2_hooks::Bypass hb2_bypass;\n"
     "        SetCompExp(hb2_ph, totalCategs > 1 ? categID : -1);\n"
     "        reuse_exponentials();\n"
     "        return false;\n"
     "      }\n",
     "RecomputeMatrix: after the parameter write-back block (calcnode.cpp:667)"),
    ("core/calcnode.cpp", "    compExp = m->Exponentiate(1., true, *store_exp_here);", ("before", -1),
     "  if (_Matrix *hb2_keep = hb2_hooks::intercept(this, m, hb2_cat, do_exponentiation, *store_exp_here)) {   // hyphy_b200\n"
     "    compExp = hb2_keep;\n"
     "    if (do_exponentiation) reuse_exponentials();\n"
     "    *store_exp_here = compExp;\n"
     "    return;\n"
     "  }\n",
     "SetCompExp: the engine exponentiates (calcnode.cpp:730)"),
]


def apply(src_root: str) -> None:
    by_file: dict[str, list] = {}
    for h in HOOKS:
        by_file.setdefault(h[0], []).append(h)
    for rel, hooks in by_file.items():
        path = os.path.join(src_root, rel)
        lines = open(path).read().split("\n")
        # resolve all insertion points against the ORIGINAL text, then insert bottom-up
        points = []
        for _, anchor, where, text, note in hooks:
            hits = [i for i, ln in enumerate(lines) if anchor in ln]
            if len(hits) != 1:
                sys.exit(f"apply_hooks: anchor for '{note}' found {len(hits)} times in {rel}: {anchor!r}")
            shift = 0
            if isinstance(where, tuple):
                where, shift = where
            at = hits[0] + (1 if where == "after" else 0) + shift
            points.append((at, text))
        for at, text in sorted(points, key=lambda x: -x[0]):
            lines[at:at] = text.rstrip("\n").split("\n")
        open(path, "w").write("\n".join(lines))
        print(f"apply_hooks: {rel}: {len(hooks)} insertion(s)")


def _writable(root: str) -> None:
    """The reference tree may be read-only: its copies must not be, or they could be neither patched nor replaced."""
    for d, _, files in os.walk(root):
        os.chmod(d, 0o755)
        for f in files:
            os.chmod(os.path.join(d, f), 0o644)


def _fresh_copy(src: str, dst: str) -> None:
    if os.path.isdir(dst):
        _writable(dst)
        shutil.rmtree(dst)
    shutil.copytree(src, dst, copy_function=shutil.copyfile)
    _writable(dst)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref", required=True)
    ap.add_argument("--out", default=os.path.join(os.path.dirname(HERE), "oracle", "_ref", "host"))
    args = ap.parse_args()
    src = os.path.join(args.out, "src")
    os.makedirs(args.out, exist_ok=True)
    _fresh_copy(os.path.join(args.ref, "src"), src)
    apply(src)
    # the reference's own batch-file library and regression tests, so that the patched binary can run them on the GPU box
    for sub, dst in (("res", "res"), ("tests/hbltests", "hbltests")):
        _fresh_copy(os.path.join(args.ref, sub), os.path.join(args.out, dst))


if __name__ == "__main__":
    main()
