"""CPU suite: tests/branch_rows_reference.py, the reference of tests/test_gpu_branch_rows.py, and the reference binary's
pinned fixture.

The brute force (every branch pinned by replacing its matrix) satisfies sum_k w_k exp(l_{b,k}) = exp(l_s) on every branch
and equals the plain mixture reference called with one-hot weights; the outside-pass restatement equals the brute force;
and -- what makes the GPU tests able to see a kernel bug at all -- each plausible bug of MUTATIONS, restated on the
outside pass, moves a row of the GPU file's own workloads by more than the tolerance that file holds the engine to."""
import math
import os

import numpy as np
import pytest

from tests import batch_reference as br
from tests import branch_rows_reference as brr
from tests import golden_cases as gc
from tests import test_gpu_branch_rows as G
from tests import test_gpu_branch_rows_shapes as GS
from tests.test_gpu_batch_mixture import meme_sets
from tests.test_gpu_shapes import TREES, flat_tree, tree_workload


def small_case(shape, K=3, n=2, seed=0):
    """A small workload (the 8-taxon codon fixture with ambiguity, or a tree shape of the shapes suite) with MEME sets."""
    if shape == "mg94_8x60_c4_ambig":
        w, _ = gc.load(shape)
    else:
        w = tree_workload(flat_tree(TREES[shape], mean_t=0.2, seed=len(shape)), 61, 60, seed=9)
    rng = np.random.default_rng(seed + len(shape))
    branch_k, V, W, _ = meme_sets(w, K, n, rng)
    pats = rng.choice(w.S, n, replace=False)
    if len(w.ambig):
        pats[0] = np.nonzero((w.leaf_states < 0).any(axis=0))[0][0]
    return w, branch_k, V, W, pats


SHAPES = ["mg94_8x60_c4_ambig", "poly7", "all_internal"]


@pytest.mark.parametrize("shape", SHAPES)
def test_brute_rows_mix_back_to_the_site(shape):
    w, branch_k, V, W, pats = small_case(shape)
    ex = G.CodonExpm(w, True)
    off = G.offsets(branch_k)
    for i, p in enumerate(pats):
        col = w.leaf_states[:, p]
        rows = brr.brute_rows(w.tree, ex, V[i], W[i], branch_k, col, w.ambig, w.pi)
        site = brr.site_ld(w.tree, ex, V[i], W[i], branch_k, col, w.ambig, w.pi)
        for b in range(len(branch_k)):
            mixed = sum(br.LD(W[i, r]) * np.exp(rows[r]) for r in range(off[b], off[b + 1]))
            assert abs(float(np.log(mixed) - site)) <= 1e-15, (b, float(np.log(mixed)), float(site))
        # a one-component branch gives the site itself
        for b in np.nonzero(branch_k == 1)[0]:
            assert abs(float(rows[off[b]] - site)) <= 1e-15


@pytest.mark.parametrize("shape", SHAPES)
def test_brute_rows_equal_one_hot_mixture_reference(shape):
    w, branch_k, V, W, pats = small_case(shape, seed=1)
    ex = G.CodonExpm(w, True)
    hot = G.one_hot(branch_k, W)
    R = W.shape[1]
    for i, p in enumerate(pats):
        col = w.leaf_states[:, p]
        rows = brr.brute_rows(w.tree, ex, V[i], W[i], branch_k, col, w.ambig, w.pi)
        for r in range(R):
            want = brr.site_ld(w.tree, ex, V[i], hot[i * R + r], branch_k, col, w.ambig, w.pi)
            assert rows[r] == want


@pytest.mark.parametrize("shape", SHAPES)
def test_outside_pass_equals_brute_force(shape):
    w, branch_k, V, W, pats = small_case(shape, seed=2)
    ex = G.CodonExpm(w, True)
    for i, p in enumerate(pats):
        col = w.leaf_states[:, p]
        a = brr.brute_rows(w.tree, ex, V[i], W[i], branch_k, col, w.ambig, w.pi)
        b = brr.outside_rows(w.tree, ex, V[i], W[i], branch_k, col, w.ambig, w.pi)
        assert np.abs((a - b) / a).max() <= 1e-16


COMPACT = [(33, False), (64, False), (48, True)]


@pytest.mark.parametrize("D,reversible", COMPACT, ids=[f"{d}{'' if r else '-nonrev'}" for d, r in COMPACT])
def test_outside_pass_on_compact_templates(D, reversible):
    """The GPU shapes file's sweep workloads (branchK 1..4, ambiguity rows, a Dirichlet root vector): the outside pass
    equals the brute force, every branch mixes back to the site, and a one-component branch gives the site."""
    case, ex = GS.sweep_rows_case(D, reversible)
    assert not np.allclose(case.root, brr.stationary(case.tmpl).astype(np.float64))
    off = G.offsets(case.branch_k)
    for s in range(4):
        args = (case.w.tree, ex, case.V[s], case.W[s], case.branch_k, case.w.leaf_states[:, case.pats[s]], case.w.ambig,
                case.root)
        a = brr.brute_rows(*args)
        assert np.abs((brr.outside_rows(*args) - a) / a).max() <= 1e-16
        site = brr.site_ld(*args)
        for b in range(len(case.branch_k)):
            mixed = sum(br.LD(case.W[s, r]) * np.exp(a[r]) for r in range(off[b], off[b + 1]))
            assert abs(float(np.log(mixed) - site)) <= 1e-15, (s, b)
        for b in np.nonzero(case.branch_k == 1)[0]:
            assert abs(float(a[off[b]] - site)) <= 1e-15


def test_pinned_fixture_is_consistent():
    """The reference binary's pinned values: the input is the workload the GPU file builds, its unpinned sites are the
    bsrel_12x80_k3 fixture's bit for bit (local weights change nothing), and every branch mixes back to its sites."""
    w, g0 = gc.load("bsrel_12x80_k3")
    g = np.load(os.path.join(gc.GOLDEN_DIR, "bsrel_12x80_k3_pinned.npz"))
    assert str(g["checksum"]) == gc.checksum(w)
    assert np.array_equal(g["site_lnL"], g0["site_lnL"]) and float(g["lnL"]) == g0["lnL"]
    wts = np.asarray(w.meta["mixture"]["weights"])
    pinned = g["pinned"].reshape(w.tree.n_branches, len(wts), -1)
    mixed = np.log((wts[None, :, None] * np.exp(pinned)).sum(axis=1))
    assert np.abs(mixed - g["site_lnL"][None]).max() <= 1e-12
    assert np.abs(pinned - g["site_lnL"][None, None]).max() > 1.0           # pinning moves the sites


# ---------------------------------------------------------------------------------------------------------------------
# mutations: each plausible kernel bug moves a row of a GPU file's workload beyond that file's tolerance
# ---------------------------------------------------------------------------------------------------------------------
def _codon(make):
    """A codon workload's first set: (outside_rows arguments, tests/test_gpu_branch_rows.py's tolerance)."""
    def case():
        w, branch_k, V, W, pats = make()
        return (w.tree, G.CodonExpm(w, False), V[0], W[0], branch_k, w.leaf_states[:, pats[0]], w.ambig, w.pi), G.TOL
    return case


def _meme_case():
    w, _ = gc.load("c2_mg94_50x1000_c1")
    rng = np.random.default_rng(10 * 2 + len("c2_mg94_50x1000_c1"))
    branch_k, V, W, _ = meme_sets(w, 2, 1, rng)
    return w, branch_k, V, W, rng.choice(w.S, 1)


def _shape_case(shape):
    w = tree_workload(flat_tree(TREES[shape], mean_t=0.2, seed=len(shape)), 61, 150, seed=9)
    rng = np.random.default_rng(len(shape))
    branch_k, V, W, _ = meme_sets(w, 2, 1, rng)
    return w, branch_k, V, W, rng.choice(w.S, 1)


def _sweep(D, reversible, root=None):
    """The GPU shapes file's sweep workload, first set, with its Dirichlet root vector (or `root`): (outside_rows
    arguments, that file's sweep tolerance)."""
    def case():
        c, ex = GS.sweep_rows_case(D, reversible)
        return (c.w.tree, ex, c.V[0], c.W[0], c.branch_k, c.w.leaf_states[:, c.pats[0]], c.w.ambig,
                c.root if root is None else root(c)), GS.TOL["sweep"]
    return case


MUTATION_CASES = {                  # mutation: a workload of one of the GPU files, and that file's tolerance
    "outside_through_P": _sweep(48, False),
    "sibling_self": _codon(_meme_case),
    "root_ones": _codon(_meme_case),
    "row_mixed": _codon(_meme_case),
    "drop_third_child": _codon(lambda: _shape_case("star40")),
    "root_stationary": _sweep(64, False),
    "message_transposed": _sweep(33, False),
    "outside_component0": _sweep(48, True),
}


def test_every_mutation_has_a_case():
    assert set(MUTATION_CASES) == set(brr.MUTATIONS)


def _shift(mutation, args):
    ref = brr.outside_rows(*args).astype(np.float64)
    mut = brr.outside_rows(*args, mutate=(mutation,)).astype(np.float64)
    with np.errstate(invalid="ignore"):
        err = np.abs(mut - ref) / np.abs(ref)
    return float(np.where(np.isnan(err), np.inf, err).max())


@pytest.mark.parametrize("mutation", list(MUTATION_CASES))
def test_mutation_moves_a_row_beyond_tolerance(mutation):
    args, tol = MUTATION_CASES[mutation]()
    ref = brr.outside_rows(*args).astype(np.float64)
    assert np.array_equal(ref, brr.outside_rows(*args, mutate=()).astype(np.float64))      # unmutated, nothing moves
    shift = _shift(mutation, args)
    print(f"{mutation}: largest relative shift {shift:.2e} against tolerance {tol:.0e}")
    assert shift > 10 * tol or math.isinf(shift), (mutation, shift)


def test_root_stationary_is_hidden_by_a_reversible_stationary_root():
    """Why workloads with root = pi on reversible models cannot see the bug: there the root vector is the template's
    stationary vector, and the mutation moves no row by a single bit."""
    c, _ = GS.sweep_rows_case(48, True)
    Q = br.dense(c.tmpl, c.tmpl.base)
    assert np.abs(c.tmpl.cf @ Q).max() <= 1e-14 * np.abs(Q).max()                   # cf is stationary
    args, _ = _sweep(48, True, root=lambda c: c.tmpl.cf)()
    assert _shift("root_stationary", args) == 0.0
