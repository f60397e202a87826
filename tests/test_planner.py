"""CPU suite: the host-side planner of the tensor-core pruning pass (hb2_plan_walk: the tree parser, dirty-node closure
and planner that hb2_create and hb2_evaluate run before they launch prune64_tc_walk_kernel).  The kernel trusts the plan blindly -- a lane waits for another lane's tile only
where the plan says WAIT, takes registers where it says CHAIN -- so the plan's invariants are checked here for many
trees, lane counts and dirty sets, and each plan is executed by a small in-order-lane simulator to prove that its
cross-lane waits cannot deadlock."""
import numpy as np
import pytest

from hyphy_b200 import engine, synth
from hyphy_b200.engine import STEP_WAIT, STEP_CHAIN, STEP_MUL, STEP_ID_MASK, STEP_FIRST, STEP_LAST


def caterpillar(n):
    """((((a,b),c),d),...) unrooted: trifurcating root.  Leaves 0..n-1, internals in post-order, root last."""
    L, I = n, n - 2
    par = np.full(L + I, -1, dtype=np.int64)
    par[0] = par[1] = 0
    for k in range(1, I):
        par[L + k - 1] = k          # previous internal hangs under the next one
        par[k + 1] = k              # with one more leaf
    par[n - 1] = I - 1              # the root gets a third child
    return par, L


def balanced(depth):
    """Complete binary tree with 2^depth leaves (root bifurcating)."""
    L = 2 ** depth
    I = L - 1
    par = np.full(L + I, -1, dtype=np.int64)
    level = list(range(L))          # flat ids of the current level
    nxt = 0
    while len(level) > 1:
        up = []
        for a, b in zip(level[::2], level[1::2]):
            par[a] = par[b] = nxt
            up.append(L + nxt)
            nxt += 1
        level = up
    return par, L


def trees():
    out = [("caterpillar12", *caterpillar(12)), ("caterpillar60", *caterpillar(60)), ("balanced6", *balanced(6))]
    for n, seed in ((8, 1), (50, 2), (200, 20260924), (333, 5)):
        t = synth.random_tree(n, seed=seed) if hasattr(synth, "random_tree") else synth.codon_workload(n, 8, 1, seed=seed).tree
        out.append((f"random{n}", np.asarray(t.flat_parents, dtype=np.int64), t.n_leaves))
    return out


TREES = trees()


def check_plan(par, L, update, lanes, split, canonical=False):
    I = len(par) - L
    ls, st = engine.plan_walk(par, L, update, lanes, split, canonical)
    children = [[] for _ in range(I)]
    for n in range(L + I - 1):
        children[par[n]].append(n)
    # expected dirty set: parents of the updated nodes and their ancestors (everything when update is None)
    dirty = np.zeros(I, dtype=bool)
    if update is None:
        dirty[:] = True
    else:
        for n in update:
            p = par[n]
            while p >= 0 and not dirty[p]:
                dirty[p] = True
                p = par[L + p]
    assert ls[0] == 0 and np.all(np.diff(ls) >= 0) and ls[-1] == len(st)
    # ---- jobs: contiguous FIRST..LAST runs; every dirty node exactly once; side jobs only for split nodes -------------
    jobs = {}                                      # slot -> (lane, order in lane, [(child, flags)])
    for r in range(lanes):
        order = 0
        i = ls[r]
        while i < ls[r + 1]:
            slot = st[i, 1] & STEP_ID_MASK
            assert st[i, 1] & STEP_FIRST, "job must start with FIRST"
            items = []
            while True:
                assert (st[i, 1] & STEP_ID_MASK) == slot
                items.append((int(st[i, 0] & STEP_ID_MASK), int(st[i, 0])))
                last = bool(st[i, 1] & STEP_LAST)
                i += 1
                if last:
                    break
                assert not (st[i, 1] & STEP_FIRST)
            assert slot not in jobs, "job scheduled twice"
            jobs[slot] = (r, order, items)
            order += 1
    assert sorted(s for s in jobs if s < I) == list(np.nonzero(dirty)[0])
    for slot, (r, order, items) in jobs.items():
        n = slot if slot < I else slot - I
        assert dirty[n]
        if slot >= I:
            assert (n in jobs) and any(f & STEP_MUL and c == L + slot for c, f in jobs[n][2]), "orphan side product"
    for n in np.nonzero(dirty)[0]:
        got = [c for c, f in jobs[n][2] if not f & STEP_MUL]
        mul = [c for c, f in jobs[n][2] if f & STEP_MUL]
        if mul:
            assert split and lanes > 1 and mul == [L + I + n] and (I + n) in jobs
            got += [c for c, f in jobs[I + n][2]]
            assert all(not f & STEP_MUL for c, f in jobs[I + n][2])
            assert sum(1 for c in children[n] if c >= L) >= 2
        else:
            assert (I + n) not in jobs
        assert sorted(got) == sorted(children[n]), "every child contracted exactly once"
    # ---- flags: CHAIN = produced by the lane's previous job; WAIT = produced by another lane in this pass -------------
    lane_jobs = {r: sorted((o, s) for s, (rr, o, _) in jobs.items() if rr == r) for r in range(lanes)}
    n_wait = 0
    for slot, (r, order, items) in jobs.items():
        for k, (c, f) in enumerate(items):
            if c < L:
                assert not f & (STEP_WAIT | STEP_CHAIN | STEP_MUL)
                continue
            prod = c - L                                            # job slot that produces this operand
            if f & STEP_CHAIN:
                assert k == 0 and order > 0 and lane_jobs[r][order - 1][1] == prod and not f & STEP_WAIT
            elif prod in jobs:                                      # produced in this pass
                pr, po, _ = jobs[prod]
                assert bool(f & STEP_WAIT) == (pr != r)
                if pr == r:
                    assert po < order
                n_wait += pr != r
            else:
                assert not f & STEP_WAIT and not dirty[prod if prod < I else prod - I] or prod >= I
    if lanes == 1:
        assert n_wait == 0
    # ---- execution: in-order lanes, a WAIT step blocks until its producer job has finished -> must terminate -----------
    pos = {r: 0 for r in range(lanes)}
    done = set()
    progressed = True
    while progressed:
        progressed = False
        for r in range(lanes):
            while pos[r] < len(lane_jobs[r]):
                slot = lane_jobs[r][pos[r]][1]
                if any((f & STEP_WAIT) and (c - L) not in done for c, f in jobs[slot][2]):
                    break
                done.add(slot)
                pos[r] += 1
                progressed = True
    assert len(done) == len(jobs), "plan deadlocks"
    return ls, st, jobs


@pytest.mark.parametrize("name,par,L", TREES, ids=[t[0] for t in TREES])
@pytest.mark.parametrize("lanes", [1, 2, 4, 8, 15])
@pytest.mark.parametrize("split", [False, True])
def test_full_tree_plan(name, par, L, lanes, split):
    check_plan(par, L, None, lanes, split)


@pytest.mark.parametrize("name,par,L", TREES, ids=[t[0] for t in TREES])
def test_partial_update_plans(name, par, L):
    rng = np.random.default_rng(7)
    I = len(par) - L
    for lanes in (1, 4, 8):
        for _ in range(6):
            k = int(rng.integers(1, 4))
            update = [int(x) for x in rng.integers(0, L + I - 1, size=k)]
            ls, st, jobs = check_plan(par, L, update, lanes, True)
            # the root is always re-pruned when anything changed
            assert (I - 1) in jobs


def test_spine_keeps_registers_and_side_products_leave_it():
    """Caterpillar = pure spine: with one lane every internal child is handed over in registers; with several lanes and a
    tree whose spine nodes have internal siblings, those siblings' contractions move into side products."""
    par, L = caterpillar(40)
    ls, st, jobs = check_plan(par, L, None, 1, True)
    chains = sum(1 for s, (_, _, items) in jobs.items() for c, f in items if f & STEP_CHAIN)
    assert chains == len(par) - L - 1                     # every internal node but the first continues a chain
    w = synth.codon_workload(200, 8, 1)
    par, L = np.asarray(w.tree.flat_parents, dtype=np.int64), w.tree.n_leaves
    _, st_split, jobs_split = check_plan(par, L, None, 8, True)
    _, st_plain, jobs_plain = check_plan(par, L, None, 8, False)
    assert any(s >= len(par) - L for s in jobs_split) and not any(s >= len(par) - L for s in jobs_plain)
    assert len(st_split) == len(st_plain) + sum(1 for s in jobs_split if s >= len(par) - L)   # one MUL step per side product


@pytest.mark.parametrize("name,par,L", TREES, ids=[t[0] for t in TREES])
@pytest.mark.parametrize("lanes", [1, 3, 8])
def test_canonical_rule_for_multifurcations(name, par, L, lanes):
    """fp64 lanes kernel: a node with more than two children is never split or chained and its children come in tree order
    (one association of the product in every plan); all other invariants hold; binary nodes may still split / chain."""
    I = len(par) - L
    children = [[] for _ in range(I)]
    for n in range(L + I - 1):
        children[par[n]].append(n)
    rng = np.random.default_rng(3)
    for update in (None, [int(x) for x in rng.integers(0, L + I - 1, size=3)]):
        ls, st, jobs = check_plan(par, L, update, lanes, True, canonical=True)
        for slot, (r, order, items) in jobs.items():
            n = slot if slot < I else slot - I
            if len(children[n]) > 2:
                assert slot < I and (I + n) not in jobs
                assert [c for c, f in items] == children[n]
                assert not any(f & (STEP_CHAIN | STEP_MUL) for c, f in items)


def test_planner_rejects_bad_input():
    par, L = caterpillar(6)
    with pytest.raises(engine.EngineError):
        engine.plan_walk(par, L, None, 0)
    with pytest.raises(engine.EngineError):
        engine.plan_walk(par, L, [99], 2)
    bad = par.copy()
    bad[L] = 0                                            # an internal node that is its own ancestor
    with pytest.raises(engine.EngineError):
        engine.plan_walk(bad, L, None, 2)
    # the tree checks hb2_create makes: one root, and it is the last node; no internal node without children
    I = len(par) - L
    two_roots = par.copy()
    two_roots[0] = -1                                     # a leaf without a parent
    root_not_last = par.copy()
    root_not_last[L + I - 2], root_not_last[L + I - 1] = -1, I - 2   # the root's last child takes its place
    childless = par.copy()
    childless[0] = childless[1] = 1                       # internal node 0 loses both its leaves
    for tree, why in ((two_roots, "root must be the last node"), (root_not_last, "root must be the last node"),
                      (childless, "internal node 0 has no children")):
        with pytest.raises(engine.EngineError, match=why):
            engine.plan_walk(tree, L, None, 2)
