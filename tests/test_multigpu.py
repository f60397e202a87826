"""GPU suite, multi-rank: one process per GPU over the engine's NCCL communicator.  Needs >= 2 visible GPUs
(`gpurun --gpus 2 -- python -m pytest tests/test_multigpu.py -m gpu`); on a single-GPU box the tests are skipped -- the
world_size-2 host logic is covered on CPU by tests/test_multirank_cpu.py."""
import json
import os
import subprocess
import sys

import pytest

from hyphy_b200 import engine

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _world():
    n = engine.device_count()
    return 8 if n >= 8 else 4 if n >= 4 else 2 if n >= 2 else 0


def _run_worker(name):
    world = _world()
    if world < 2:
        pytest.skip("needs at least 2 GPUs")
    port = 29500 + (os.getpid() % 400)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "tests", "multigpu_worker.py"), name]
    pr = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900, cwd=ROOT)
    lines = [l for l in pr.stdout.splitlines() if l.startswith("MULTIGPU ")]
    assert lines, pr.stdout[-3000:]
    res = json.loads(lines[-1][len("MULTIGPU "):])
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    with open(os.path.join(ROOT, "gpurun_out", "multigpu_parity.jsonl"), "a") as f:
        f.write(json.dumps(res) + "\n")
    assert pr.returncode == 0, res
    assert all(r["ok_all_ranks"] for r in res["layouts"]), res


@pytest.mark.parametrize("name", ["mg94_30x100_c4_ambig", "mg94_200x64_c4_scaling", "ns_mg94_200x2000_c4"])
def test_sharded_layouts_match_reference_golden(name, engine_lib):
    _run_worker(name)


def test_class_groups_ignore_zero_weight_class(engine_lib):
    """Two class groups, the group of the highest class with weight 0: the other group's classes must not be flushed."""
    _run_worker("class_groups_zero_weight")
