"""GPU suite (pytest -m gpu): the tensor walk kernel runs two pattern tiles of one class per CTA, one per warpgroup.

A unit is two tiles or, at an odd tile count (and where the host fills idle SMs with single tiles), one; the second
warpgroup of a single-tile unit idles but the two share one staging ring.  Covered here against the oracle:
  * tile counts T = 1, 2, 3 (T = 1 and 3 leave one unit half empty): likelihoods, a pinned node, partial updates;
  * one lane per unit with more units than resident CTAs, so a CTA loops over several units of different sizes;
  * pairing touches no per-pattern arithmetic: a pattern's likelihood and scaling exponent are bit-identical whether the
    engine holds the first 128, 256 or 384 patterns of one alignment."""
import numpy as np
import pytest

from hyphy_b200 import synth, LikelihoodFunction, engine
from tests.test_gpu_shapes import tree_workload, oracle_P, check_lnl, check_forced, check_partial

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _need_gpu(engine_lib):
    assert engine.device_count() > 0, "GPU tests need a CUDA device (no fallback exists)"


def prefix(n):
    """The first n distinct patterns of one 61-state alignment on a 40-leaf tree (1 500 distinct patterns in all)."""
    return tree_workload(synth.random_tree(40, 5, mean_t=0.2), 61, 1500, seed=9, n_patterns=n)


@pytest.mark.parametrize("S", [100, 256, 300])
def test_half_empty_and_full_units(S):
    """S = 100 (T = 1) and 300 (T = 3) leave one unit with an idle warpgroup; S = 256 is one full pair."""
    w = prefix(S)
    L = w.tree.n_leaves
    P = oracle_P(w)
    lf = LikelihoodFunction(w, flags=engine.FLAG_DEFAULT)
    assert lf.part.pruning_kernel == "prune64_tc_walk_kernel"
    lf.set_all_matrices()
    check_lnl(lf, w, "tc", P)
    inner = L + w.tree.n_internal // 2
    check_forced(lf, w, "tc", [inner], P=P)
    check_partial(lf, w, "tc", 3, P)
    check_partial(lf, w, "tc", inner, P)
    lf.close()


def test_one_lane_loops_over_units(monkeypatch):
    """HB2_WALK_LANES=1, 4 classes, 8 832 patterns: T = 69 tiles per class is odd and the units (a pair or a single tile)
    outnumber the CTAs an H100 holds, so a CTA walks several units in turn."""
    monkeypatch.setenv("HB2_WALK_LANES", "1")
    w = synth.codon_workload(12, 9000, 4, seed=31, mean_t=0.5)
    assert w.S > 68 * 128
    lf = LikelihoodFunction(w, flags=engine.FLAG_DEFAULT)
    lf.set_template()
    lf.set_all_compiled()
    check_lnl(lf, w, "tc")
    check_partial(lf, w, "tc", 2)
    lf.close()


@pytest.mark.parametrize("lanes", ["1", "2", "4"])
def test_pairing_leaves_per_pattern_results_alone(lanes, monkeypatch):
    """At a fixed lane count every pattern runs the same steps with the same operands, whichever unit holds its tile.
    At 2 and 4 lanes the tiles of T = 2 and 3 are paired.  At one lane the host gives every tile of these one-class
    workloads a CTA of its own (the units are split back into single tiles to fill the SMs): that covers the split path."""
    monkeypatch.setenv("HB2_WALK_LANES", lanes)
    sites = {}
    for n in (128, 256, 384):
        w = prefix(n)
        lf = LikelihoodFunction(w, flags=engine.FLAG_DEFAULT)
        lf.set_all_matrices()
        check_lnl(lf, w, "tc", oracle_P(w))
        _, sl, ss = lf.compute(want_sites=True)
        sites[n] = (sl, ss)
        lf.close()
    for n in (128, 256):
        assert np.array_equal(sites[n][0], sites[384][0][:n]), n
        assert np.array_equal(sites[n][1], sites[384][1][:n]), n
