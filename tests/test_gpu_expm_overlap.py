"""GPU suite: the 64-state shared-powers expm stage with its power tables built on the partition's side stream while the
classification runs, and with the finishing kernel working from the list of entries the earlier stages leave to it.
Covers one batch that rebuilds some groups' tables while other groups' entries are classified against their cached
directions, finishing lists that are empty and non-empty in consecutive batches (shift-0 entries next to entries that
need squarings, NaN input and unflagged entries), lengths that are no multiple of the polynomial kernel's chunk, and two
partitions evaluated back to back."""
import numpy as np
import pytest

from hyphy_b200 import LikelihoodFunction, engine
from oracle import port
from tests import golden_cases as gc

pytestmark = pytest.mark.gpu

FLAGS = pytest.mark.parametrize("flags", [engine.FLAG_FORCE_FP64, engine.FLAG_DEFAULT], ids=["fp64", "tc"])


@pytest.fixture(scope="module", autouse=True)
def _need_gpu(engine_lib):
    assert engine.device_count() > 0, "GPU tests need a CUDA device (no fallback exists)"


def small_rates(Qt):
    """Qt with every class scaled so that no matrix needs squarings (||Q t||_inf <= 2 < 2.3): every entry of a batch of
    these is finished by the polynomial kernel and the finishing list stays empty."""
    Qs = Qt.copy()
    for c in range(Qs.shape[0]):
        Qs[c] *= 2.0 / np.abs(Qs[c]).sum(axis=2).max()
    return Qs


def check(lf, expected, nan=()):
    for (c, b), Q in expected.items():
        P = lf.part.read_transition(c, b)
        if (c, b) in nan:
            assert np.all(np.isnan(P)), (c, b)
            continue
        np.testing.assert_allclose(P, port.expm(Q, True), rtol=0, atol=3e-14, err_msg=f"class {c} branch {b}")
        assert np.all(P >= 0) and np.abs(P.sum(axis=1) - 1.0).max() <= 1e-14, (c, b)


@FLAGS
def test_rebuilt_and_cached_groups_in_one_batch(flags):
    w, _ = gc.load("mg94_30x100_c4_ambig")
    nb, C = w.tree.n_branches, w.C
    Qs = small_rates(w.Qt())
    lf = LikelihoodFunction(w, flags=flags)
    expected = {}
    # batch 1: every group rebuilt, every entry shift 0 -> empty finishing list
    for c in range(C):
        lf.part.set_matrices(c, lf.all_nodes, Qs[c])
        expected.update({(c, b): Qs[c, b] for b in range(nb)})
    assert (C * nb) % 16 != 0
    check(lf, expected)
    # batch 2: class 0 rebuilt (all branches: one needs squarings, one is NaN); classes 1 and 2 classified against the
    # directions batch 1 left (a few branches each: scaled copies, one needing squarings, one not a multiple)
    Q0 = Qs[0].copy()
    Q0[3] *= 60.0
    Q0[5] = np.nan
    lf.part.set_matrices(0, lf.all_nodes, Q0)
    expected.update({(0, b): Q0[b] for b in range(nb)})
    b1 = np.array([1, 4, 8, 9, 12], dtype=np.int64)
    Q1 = Qs[1, b1] * 1.1
    Q1[2] *= 25.0
    Q1[4] = Qs[2, 12]                                           # another class's direction: unflagged, general path
    lf.part.set_matrices(1, b1, Q1)
    expected.update({(1, int(b)): Q1[i] for i, b in enumerate(b1)})
    b2 = np.array([0, 7, 20], dtype=np.int64)
    Q2 = Qs[2, b2] * 0.5
    lf.part.set_matrices(2, b2, Q2)
    expected.update({(2, int(b)): Q2[i] for i, b in enumerate(b2)})
    assert (nb + len(b1) + len(b2)) % 16 != 0
    check(lf, expected, nan={(0, 5)})
    # batch 3: the list of batch 2 was emptied; all shift 0 again
    for c in range(C):
        lf.part.set_matrices(c, lf.all_nodes, Qs[c] * 0.9)
        expected.update({(c, b): Qs[c, b] * 0.9 for b in range(nb)})
    check(lf, expected)
    lf.close()


@FLAGS
def test_two_partitions_back_to_back(flags):
    w, g = gc.load("mg94_30x100_c4_ambig")
    nb, C = w.tree.n_branches, w.C
    Qt = w.Qt()
    Qt2 = Qt.copy()
    Qt2[:, ::3] *= 30.0                                         # every third branch needs squarings
    lfa, lfb = LikelihoodFunction(w, flags=flags), LikelihoodFunction(w, flags=flags)
    for c in range(C):
        lfa.part.set_matrices(c, lfa.all_nodes, Qt[c])
        lfb.part.set_matrices(c, lfb.all_nodes, Qt2[c])
    la, lb = lfa.compute(), lfb.compute()
    rtol = 1e-10 if flags == engine.FLAG_FORCE_FP64 else 1e-7
    assert abs(la - g["lnL"]) <= rtol * abs(g["lnL"]), (la, g["lnL"])
    ref_b, _ = port.lnl(w, Qt=Qt2)
    assert abs(lb - ref_b) <= rtol * abs(ref_b), (lb, ref_b)
    for it in range(3):                                         # replays interleaved: each partition forks its own side stream
        _, _, ra = lfa.part.time_resident(w.class_weights, w.pi, iters=2)
        _, _, rb = lfb.part.time_resident(w.class_weights, w.pi, iters=2)
        assert abs(ra - la) <= 1e-12 * abs(la) and abs(rb - lb) <= 1e-12 * abs(lb), (it, ra, la, rb, lb)
    check(lfa, {(c, b): Qt[c, b] for c in range(C) for b in range(nb)})
    check(lfb, {(c, b): Qt2[c, b] for c in range(C) for b in range(nb)})
    lfa.close()
    lfb.close()
