"""CPU suite: the patched host binary (oracle/_ref/host/hyphy, built by __graft_entry__.build() where the reference sources exist)
without a GPU -- what must keep working, and what must fail loudly.  Skipped when the binary is not there."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

from oracle import ref_harness as rh
from tests import golden_cases as gc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "oracle", "_ref", "host")
HOST_BIN = os.path.join(BUILD, "hyphy")

pytestmark = pytest.mark.skipif(not os.path.isfile(HOST_BIN), reason="patched host binary not built (needs the reference sources)")


def _no_gpu_env(**extra):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", **extra)       # also on a GPU box: these tests are about the no-device paths
    return env


def test_engine_off_is_the_unmodified_cpu_path():
    """HYPHY_B200=0: the hooks are inert and the patched binary reproduces the unmodified binary's fixture."""
    w, g = gc.load("mg94_8x60_c1")
    r = rh.run_reference(w, binary=HOST_BIN, env_extra={"HYPHY_B200": "0", "CUDA_VISIBLE_DEVICES": ""})
    assert abs(r["lnL"] - g["lnL"]) <= 1e-12 * abs(g["lnL"])
    assert np.abs(r["site_lnL"] - g["site_lnL"]).max() <= 1e-9
    assert not r["engine"]


def test_engine_on_without_a_gpu_fails_loudly():
    """No CPU fallback once a partition is handed to the engine: the run must abort with a message, not compute on the host."""
    w, _ = gc.load("mg94_8x60_c1")
    with pytest.raises(Exception) as e:
        rh.run_reference(w, binary=HOST_BIN, env_extra={"CUDA_VISIBLE_DEVICES": ""})
    assert "CUDA" in str(e.value) or "hyphy_b200" in str(e.value) or "device" in str(e.value)


def test_two_sequence_analysis_stays_on_the_host_path():
    """likefunc.cpp:11260-11281: two-sequence likelihood functions have no internal-node cache and never reach the pruning
    branch; the hook must leave them alone -- the reference's own TwoSequenceTest.bf passes with the engine enabled and no GPU."""
    test = os.path.join(BUILD, "hbltests", "SimpleOptimizations", "TwoSequenceTest.bf")
    if not os.path.isfile(test):
        pytest.skip("hbltests not copied")
    from host import regress
    work = regress.work_tree()
    test = os.path.join(work, "hbltests", "SimpleOptimizations", "TwoSequenceTest.bf")
    tmp = tempfile.mkdtemp(prefix="hb2two_")
    pr = subprocess.run([HOST_BIN, f"LIBPATH={os.path.join(work, 'res')}", test], cwd=tmp, stdin=subprocess.DEVNULL,
                        stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=_no_gpu_env(), timeout=300)
    assert pr.returncode == 0 and "[TEST PASSED]" in pr.stdout, pr.stdout[-800:]
