"""GPU suite (pytest -m gpu): the tensor walk kernel's contraction D^T[parents][patterns] = P * X^T (one
wgmma.m64n128k8 per k-step and product) and the read-back of its accumulator fragments, against the oracle.

  * Without anchors (HB2_ANCHOR_THR=2.0: every entry of a row is below the threshold) the whole contraction runs on the
    tensor core, so every parent state of every pattern goes through the read-back.  Truncating fp32 accumulation then
    biases lnL by about 1e-7 relative (hb2_kernels_tc.cuh), so these cases are held to the 1e-6 contract, and each
    pattern to 1e-5 or 1e-6 of its own log-likelihood, whichever is larger: on the long-branch trees a pattern's
    log-likelihood is around -100 and its error without anchors reaches 1.8e-5.  The engine reads the threshold once
    per process, so these cases run in a subprocess (this file run as a script).
  * At the default threshold the same cases are held to the suite's tensor-path tolerances, 1e-7 and 1e-5.
  * Cases: the north-star workload against the reference's golden values; a codon workload with long branches, whose
    rows are diffuse; generic models with 33, 48, 61 and 64 states (parent rows beyond D are padding) on rooted binary
    trees with long branches, at 100, 256 and 300 patterns (1, 2 and 3 tiles: a single-tile unit, a pair, both).
  * On the rooted binary trees every node multiplies exactly two factors, so a partial evaluation reproduces the full
    one bit for bit on the tensor path too."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from hyphy_b200 import LikelihoodFunction, engine  # noqa: E402
from oracle import port  # noqa: E402
from tests import golden_cases as gc  # noqa: E402
from tests.test_gpu_shapes import flat_tree, tree_workload, oracle_P, oracle_sites, oracle_lnl, _site_lnl  # noqa: E402

pytestmark = pytest.mark.gpu

NO_ANCHORS = (1e-6, 1e-5, 1e-6)     # lnL rtol, per-pattern atol, per-pattern rtol
DEFAULT = (1e-7, 1e-5)
# (states, patterns) of the generic-model cases: tiles 1, 2, 3, 3
STATE_CASES = {"D33": (33, 100), "D48": (48, 256), "D61": (61, 300), "D64": (64, 300)}
CASES = ["north_star", "diffuse"] + list(STATE_CASES)


def binary_spec(n, rng):
    """Nested children list of a random rooted binary tree with n leaves (see flat_tree)."""
    if n == 1:
        return 0
    k = int(rng.integers(1, n))
    return [binary_spec(k, rng), binary_spec(n - k, rng)]


def workload(name):
    if name == "north_star":
        return gc.load("ns_mg94_200x2000_c4")[0]
    if name == "diffuse":
        from hyphy_b200 import synth
        return synth.codon_workload(24, 1500, 4, seed=17, mean_t=1.5)
    D, S = STATE_CASES[name]
    tree = flat_tree(binary_spec(30, np.random.default_rng(D)), mean_t=1.0, seed=D)
    return tree_workload(tree, D, S + 300, seed=3, n_patterns=S)


def partial_node(w):
    return w.tree.n_leaves + w.tree.n_internal // 2


def run_case(name):
    """lnL and per-pattern values; on the binary-tree cases also a partial and a full evaluation after one branch of
    every class changed."""
    w = workload(name)
    lf = LikelihoodFunction(w, flags=engine.FLAG_DEFAULT)
    assert lf.part.pruning_kernel == "prune64_tc_walk_kernel"
    lf.set_all_matrices()
    lnl, sl, ss = lf.compute(want_sites=True)
    out = {"lnl": lnl, "sl": sl, "ss": ss}
    if name in STATE_CASES:
        node = partial_node(w)
        w.tree.t[node] *= 1.6
        Qt = w.Qt()
        lf.part.set_matrices(0, [node], Qt[0, node:node + 1])
        out["part"], out["part_sl"], out["part_ss"] = lf.compute(update_nodes=[node], want_sites=True)
        out["full"], out["full_sl"], out["full_ss"] = lf.compute(update_nodes=None, want_sites=True)
        w.tree.t[node] /= 1.6
    lf.close()
    return out


def check(name, out, rtol, atol, site_rtol=0.0):
    """lnL within rtol of the oracle; every pattern within max(atol, site_rtol * |its log-likelihood|)."""
    w = workload(name)
    got = _site_lnl(out["sl"], out["ss"])
    if name == "north_star":
        g = gc.load("ns_mg94_200x2000_c4")[1]
        ref, site, got = g["lnL"], g["site_lnL"], got[w.site_to_pattern]
    elif name == "diffuse":
        ref, site = port.lnl(w, sparse_storage=True)
    else:
        P = oracle_P(w)
        ref, site = oracle_sites(w, P)
    assert np.isfinite(out["lnl"]) and abs(out["lnl"] - ref) <= rtol * abs(ref), (out["lnl"], ref)
    excess = np.abs(got - site) - np.maximum(atol, site_rtol * np.abs(site))
    assert excess.max() <= 0, (np.abs(got - site).max(), excess.max())
    if name in STATE_CASES:
        node = partial_node(w)
        w.tree.t[node] *= 1.6
        ref = oracle_lnl(w, w.Qt(), P, node)
        w.tree.t[node] /= 1.6
        assert abs(out["part"] - ref) <= rtol * abs(ref), (out["part"], ref)
        assert out["part"] == out["full"], (out["part"], out["full"])
        assert np.array_equal(out["part_sl"], out["full_sl"]) and np.array_equal(out["part_ss"], out["full_ss"])


@pytest.fixture(scope="module", autouse=True)
def _need_gpu(engine_lib):
    assert engine.device_count() > 0, "GPU tests need a CUDA device (no fallback exists)"


@pytest.fixture(scope="module")
def no_anchor_results(tmp_path_factory):
    """Every case evaluated once by a subprocess with HB2_ANCHOR_THR=2.0."""
    d = tmp_path_factory.mktemp("walk_shape")
    env = dict(os.environ, HB2_ANCHOR_THR="2.0")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.abspath(__file__), str(d)]
    pr = subprocess.run(cmd, env=env, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1200)
    assert pr.returncode == 0, pr.stdout[-3000:]
    return {name: dict(np.load(os.path.join(d, name + ".npz"))) for name in CASES}


@pytest.mark.parametrize("name", CASES)
def test_no_anchors_whole_contraction_on_the_tensor_core(name, no_anchor_results):
    out = {k: (v.item() if v.ndim == 0 else v) for k, v in no_anchor_results[name].items()}
    check(name, out, *NO_ANCHORS)


@pytest.mark.parametrize("name", CASES)
def test_default_anchor_threshold(name):
    assert "HB2_ANCHOR_THR" not in os.environ
    check(name, run_case(name), *DEFAULT)


if __name__ == "__main__":
    from hyphy_b200 import build
    build.build()
    engine.load_library()
    for case in CASES:
        np.savez(os.path.join(sys.argv[1], case + ".npz"), **run_case(case))
