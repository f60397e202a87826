"""GPU suite: the 64-state shared-powers expm stage on batches shaped to cross its chunk and cluster boundaries.  The
polynomial kernel finishes entries that need no squaring inside one cluster per chunk (the row repair reads the other
slices' column sums); the finishing kernel strides over the whole batch and only touches entries that need squarings
or carry NaN.  One batch here holds a run of retired entries (whole chunks with nothing to do), rate-class (group)
changes inside a chunk, a length that is no multiple of the chunk, and shift-0, shift > 0 and NaN entries side by side."""
import numpy as np
import pytest

from hyphy_b200 import LikelihoodFunction, engine
from oracle import port
from tests import golden_cases as gc

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _need_gpu(engine_lib):
    assert engine.device_count() > 0, "GPU tests need a CUDA device (no fallback exists)"


@pytest.mark.parametrize("flags", [engine.FLAG_FORCE_FP64, engine.FLAG_DEFAULT], ids=["fp64", "tc"])
def test_mixed_batch_with_retired_chunks(flags):
    w, _ = gc.load("mg94_30x100_c4_ambig")
    nb, C = w.tree.n_branches, w.C
    Qt = w.Qt()
    Qt[1, 9] *= 60.0                                         # rho ~ 10: squarings after the polynomial
    Qt[1, 10] *= 4.0                                         # a few squarings
    Qt[3, 11] *= 1e-7                                        # tiny rho
    Qt[2, 4] = np.nan                                        # NaN input: a NaN matrix, the rest of the class unaffected
    lf = LikelihoodFunction(w, flags=flags)
    lf.part.set_matrices(0, lf.all_nodes, Qt[0] * 2.0)      # handed over again below: nb retired entries lead the batch
    for c in range(C):
        lf.part.set_matrices(c, lf.all_nodes, Qt[c])
    assert (nb + C * nb) % 8 != 0
    for c in range(C):
        for b in range(nb):
            P = lf.part.read_transition(c, b)
            if (c, b) == (2, 4):
                assert np.all(np.isnan(P))
                continue
            np.testing.assert_allclose(P, port.expm(Qt[c, b], True), rtol=0, atol=5e-13 if (c, b) == (1, 9) else 3e-14,
                                       err_msg=f"class {c} branch {b}")
            assert np.all(P >= 0) and np.abs(P.sum(axis=1) - 1.0).max() <= 1e-14
    lf.close()
