"""GPU suite, part 2: the REAL boundary.  oracle/_ref/host/hyphy is a build copy of the reference with the hook calls of
host/apply_hooks.py inserted and host/hb2_hyphy_hooks.cpp linked against libhyphy_b200.so (built by
__graft_entry__.build() where the reference sources exist; oracle/_ref/ is carried to the GPU machine with the tree).  The same HBL scripts that produced the golden fixtures with
the UNMODIFIED reference binary are fed to the patched binary: `LFCompute`, `ConstructCategoryMatrix`, `Optimize` now run
on the engine, behind `_LikelihoodFunction::ComputeBlock`, with no change to the batch files."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import ref_harness as rh
from tests import golden_cases as gc

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST_DIR = os.path.join(ROOT, "oracle", "_ref", "host")
HOST_BIN = os.path.join(HOST_DIR, "hyphy")
# what the UNMODIFIED reference binary printed for the evaluation stream and the ancestral reconstructions below
# (tools/make_golden.py --runs)
with open(os.path.join(ROOT, "tests", "golden", "reference_runs.json")) as _f:
    REFERENCE_RUNS = json.load(_f)
MODES = {"fp64": ({}, 1e-10, 1e-8), "tc": ({"HYPHY_B200_TC": "1"}, 1e-7, 1e-5)}     # the host's default is fp64 (see hb2_hyphy_hooks.h)


@pytest.fixture(scope="module", autouse=True)
def _need_host():
    assert os.path.isfile(HOST_BIN), f"{HOST_BIN} is missing: run __graft_entry__.build() where the reference sources exist"


def _tol(w, mode):
    if mode == "tc" and w.D > 32:
        return MODES["tc"][1:]
    return MODES["fp64"][1:]


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("name", gc.SMALL + gc.MEDIUM)
def test_patched_host_reproduces_reference_fixture(name, mode):
    """lnL (LFCompute) and per-site log-likelihoods (ConstructCategoryMatrix SITE_LOG_LIKELIHOODS, i.e. the per-class
    ComputeBlock path with siteRes / scaler counts combined by the HOST) of the patched binary against the fixture the
    unmodified binary produced from the same script."""
    w, g = gc.load(name)
    env = dict(MODES[mode][0], HYPHY_B200_VERBOSE="1")
    r = rh.run_reference(w, binary=HOST_BIN, env_extra=env)
    rtol, atol = _tol(w, mode)
    assert any("partition 0 on device" in l for l in r["engine"]), "the engine did not run this likelihood function"
    assert abs(r["lnL"] - g["lnL"]) <= rtol * abs(g["lnL"]), (r["lnL"], g["lnL"])
    assert np.abs(r["site_lnL"] - g["site_lnL"]).max() <= max(atol, 1e-9)


def test_patched_host_evaluation_stream_and_partial_updates():
    """The bench's evaluation stream (one global parameter perturbed per evaluation -> every matrix re-exponentiated on the
    device) through the patched binary: final lnL of the loop equals the unmodified binary's to 1e-7 relative."""
    a = REFERENCE_RUNS["evaluation_stream"]
    w, g = gc.load(a["case"])
    b = rh.run_reference(w, n_evals=a["n_evals"], n_warm=a["n_warm"], per_site=False, binary=HOST_BIN,
                         env_extra={"HYPHY_B200_VERBOSE": "1", "HYPHY_B200_TC": "1"})
    assert abs(b["loop_lnL"] - a["loop_lnL"]) <= 1e-7 * abs(a["loop_lnL"])
    assert abs(b["lnL"] - g["lnL"]) <= 1e-7 * abs(g["lnL"])


@pytest.mark.parametrize("name", ["mg94_8x60_c1", "mg94_8x60_c4_ambig", "c1_hky85_8x500", "mg94_30x100_c4_ambig"])
def test_patched_host_ancestral_reconstruction_matches_reference(name):
    """ReconstructAncestors (joint ML, likefunc2.cpp:308 -> tree.cpp:4209) reads the nodes' transition matrices -- and, for
    rate variation, the class assignments -- on the HOST; with the engine they are copied back from the device first
    (hb2_hooks::materialize).  Same ancestral sequences as the unmodified binary, in both precisions."""
    w, g = gc.load(name)
    ref = {"ancestors": REFERENCE_RUNS["ancestors"][name]}
    assert ref["ancestors"] and all(len(a) == len(ref["ancestors"][0]) for a in ref["ancestors"])
    for mode in MODES:
        r = rh.run_reference(w, ancestors=True, per_site=False, binary=HOST_BIN, env_extra=dict(MODES[mode][0], HYPHY_B200_VERBOSE="1"))
        assert any("partition 0 on device" in l for l in r["engine"])
        assert abs(r["lnL"] - g["lnL"]) <= _tol(w, mode)[0] * abs(g["lnL"])
        if mode == "fp64":
            assert r["ancestors"] == ref["ancestors"]
        else:       # fp32 conditionals never enter the joint reconstruction (it recomputes from the matrices), but P's last bits can flip a tie
            diff = sum(a != b for x, y in zip(r["ancestors"], ref["ancestors"]) for a, b in zip(x, y))
            assert len(r["ancestors"]) == len(ref["ancestors"]) and diff <= 2, diff


def test_patched_host_reference_ancestor_batch_file():
    """The reference's own Ancestors/NucAncestors.bf compares the joint ML reconstruction with sequences stored in the file
    ([OK: ML SEQUENCE RECONSTRUCTION]); its later sections fail with the unmodified binary as well and are not judged."""
    import tempfile
    from host import regress
    work = regress.work_tree()
    test = os.path.join(work, "hbltests", "Ancestors", "NucAncestors.bf")
    tmp = tempfile.mkdtemp(prefix="hb2anc_")
    pr = subprocess.run([HOST_BIN, f"LIBPATH={os.path.join(work, 'res')}", test], cwd=tmp, stdin=subprocess.DEVNULL,
                        stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=dict(os.environ, HYPHY_B200_VERBOSE="1"), timeout=600)
    assert "partition 0 on device" in pr.stdout
    assert "[OK: ML SEQUENCE RECONSTRUCTION]" in pr.stdout and "MISMATCHED" not in pr.stdout, pr.stdout[-1500:]


def test_patched_host_runs_reference_regression_batch_files():
    """The reference's own regression batch files (tests/hbltests: optimisations, category variables, HMM, explicit-form
    mixtures, ancestral reconstruction, per-site likelihoods) through the patched binary, UNMODIFIED: same verdict and the
    same fitted log-likelihoods as the unmodified reference binary recorded in tests/golden/hbltests_expected.json."""
    pr = subprocess.run([sys.executable, os.path.join(ROOT, "host", "regress.py"), "check"], stdout=subprocess.PIPE, text=True)
    rows = [json.loads(l) for l in pr.stdout.splitlines() if l.startswith("{")]
    assert rows, pr.stdout[-2000:]
    bad = [r for r in rows if not r["ok"]]
    assert not bad, [(r["test"], r["got"]["verdict"], r["got"]["lnL"], r["got"]["tail"][-300:]) for r in bad]
