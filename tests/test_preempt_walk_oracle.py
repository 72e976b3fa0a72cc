"""CPU: the sequential preemption walk (include/bsched.h bs_preempt_walk) on both CPU restatements,
tests/preempt_walk_ref.c and tests/pyref_preempt_walk.py: the hand-built cases of tests/preempt_walk_cases.py, the two
restatements against each other on random tables with and without PodDisruptionBudget bits and gang units, and the
walk's invariants.  The GPU is compared with the C restatement in tests/test_gpu_preempt_walk.py."""
import importlib
import itertools

import numpy as np
import pytest

import preempt_pdb_ref
import preempt_walk_cases as W
import preempt_walk_ref
import pyref_preempt_walk

S = importlib.import_module("batch-scheduler_b200.snapshot")


def _rows(r, k):
    return int(r.node[k]), r.victims_of(k), int(r.outcome[k])


def _check(snap, bound, pods, gang):
    """The C walk, checked against the Python walk and for rows evicted at most once."""
    got = preempt_walk_ref.walk(snap, bound, pods, gang)
    py, evicted_by = pyref_preempt_walk.walk(snap, bound, pods, gang)
    for k in range(len(pods)):
        node, victims, cand, outcome = py[k]
        assert (int(got.node[k]), got.victims_of(k), int(got.n_candidates[k]), int(got.outcome[k])) == \
            (node, victims, cand, outcome), k
    assert got.evicted_by.tolist() == evicted_by
    assert len(set(got.victims.tolist())) == len(got.victims)
    for k in range(len(pods)):
        assert all(got.evicted_by[v] == k for v in got.victims_of(k))
    assert (got.evicted_by >= 0).sum() == len(got.victims)
    return got


@pytest.mark.parametrize("name", sorted(W.cases()))
def test_hand_built_case(name):
    snap, bound, pods, gang, want, plain = W.cases()[name]
    got = _check(snap, bound, pods, gang)
    assert [_rows(got, k) for k in range(len(pods))] == want
    p = preempt_pdb_ref.preempt(snap, bound, pods)
    assert [(int(p.node[k]), p.victims_of(k)) for k in range(len(pods))] == plain


@pytest.mark.parametrize("seed,L,violating,gang",
                         list(itertools.product(range(8), (5, 9), (0.0, 0.5), (False, True))))
def test_c_restatement_agrees_with_pyref_random(seed, L, violating, gang):
    snap, bound = W.random_table(seed, L, violating)
    pods = W.queue(snap, gang=gang)
    got = _check(snap, bound, pods, gang)
    if not gang:
        assert ((got.outcome == W.NONE) == (got.node < 0)).all()


def test_random_tables_reach_the_walk():
    """Over the random tables, the walk differs from independent what-ifs, gangs roll back, and victims are chosen."""
    differ = rolled = victims = 0
    for seed, L in itertools.product(range(8), (5, 9)):
        snap, bound = W.random_table(seed, L, 0.5)
        pods = W.queue(snap, gang=True)
        walk = preempt_walk_ref.walk(snap, bound, pods, True)
        plain = preempt_pdb_ref.preempt(snap, bound, pods)
        differ += any((int(walk.node[k]), walk.victims_of(k)) != (int(plain.node[k]), plain.victims_of(k))
                      for k in range(len(pods)))
        rolled += int((walk.outcome == W.ROLLED_BACK).any())
        victims += len(walk.victims)
    assert differ >= 4 and rolled >= 2 and victims > 0


@pytest.mark.parametrize("seed,violating", list(itertools.product(range(6), (0.0, 0.5))))
def test_one_preemptor_is_bs_preempt(seed, violating):
    snap, bound = W.random_table(seed, 5, violating)
    for p in range(snap.pods.n):
        for gang in (False, True):
            walk = preempt_walk_ref.walk(snap, bound, [p], gang)
            want = preempt_pdb_ref.preempt(snap, bound, [p])
            assert int(walk.n_candidates[0]) == int(want.n_candidates[0])
            if walk.outcome[0] == W.ROLLED_BACK:
                assert gang and want.node[0] < 0
            else:
                assert (int(walk.node[0]), walk.victims_of(0)) == (int(want.node[0]), want.victims_of(0))


@pytest.mark.parametrize("seed", range(6))
def test_disjoint_gates_give_bs_preempt(seed):
    """Each preemptor selects one label bit and each node carries one, so no two preemptors share a candidate node:
    every step sees the uploaded state of its nodes."""
    snap, bound = W.random_table(seed, 5, 0.5, P=8, N=16)
    nt, pt = snap.nodes, snap.pods
    nt.label_mask[:] = np.uint64(1) << (np.arange(nt.n) % 8).astype(np.uint64)
    nt.taint_mask[:] = 0
    pt.sel_mask[:] = np.uint64(1) << np.arange(pt.n).astype(np.uint64)
    pods = W.queue(snap)
    walk = preempt_walk_ref.walk(snap, bound, pods)
    want = preempt_pdb_ref.preempt(snap, bound, pods)
    for k in range(len(pods)):
        assert (int(walk.node[k]), walk.victims_of(k), int(walk.n_candidates[k])) == \
            (int(want.node[k]), want.victims_of(k), int(want.n_candidates[k]))
    assert len(walk.victims) > 0


@pytest.mark.parametrize("seed", range(6))
def test_rolled_back_unit_leaves_no_trace(seed):
    """A walk A + U + B, where the gang unit U rolls back, gives A and B the answers of the walk A + B."""
    snap, bound = W.random_table(seed, 5, 0.5, P=12, G=3)
    pt = snap.pods
    pt.priority[:] = 2**31 - 1
    u = np.flatnonzero(pt.gid == 0)[:3].tolist()
    if len(u) < 2:
        u = [0, 1]
        pt.gid[u] = 0
    pt.req[0, u[-1]] = 1 << 50   # the unit's last member fits nowhere
    rest = [p for p in range(pt.n) if p not in u and pt.gid[p] < 0]
    a, b = rest[:len(rest) // 2], rest[len(rest) // 2:]
    with_u = preempt_walk_ref.walk(snap, bound, a + u + b, True)
    without = preempt_walk_ref.walk(snap, bound, a + b, True)
    assert (with_u.outcome[len(a):len(a) + len(u)] == W.ROLLED_BACK).all()
    keep = list(range(len(a))) + list(range(len(a) + len(u), len(a) + len(u) + len(b)))
    for k, j in zip(keep, range(len(a) + len(b))):
        assert _rows(with_u, k) == _rows(without, j)
        assert int(with_u.n_candidates[k]) == int(without.n_candidates[j])
    ev = with_u.evicted_by.copy()
    ev[ev >= len(a) + len(u)] -= len(u)
    np.testing.assert_array_equal(ev, without.evicted_by)


@pytest.mark.parametrize("seed", range(4))
def test_gid_past_the_group_table_is_a_unit_of_one(seed):
    """Pods whose gid is >= n_groups are units of one under gang units in both restatements, contiguous or not."""
    snap, bound = W.random_table(seed, 5, 0.5, P=10, G=3)
    pt = snap.pods
    pt.priority[:] = 2**31 - 1
    pt.gid[[0, 3, 4, 8]] = snap.groups.n + 1
    pt.req[0, 3] = 1 << 50   # fits nowhere: only its own unit rolls back
    pods = list(range(pt.n))
    got = _check(snap, bound, pods, True)
    assert preempt_walk_ref.units_last(snap, pods, True)[[0, 3, 4, 8]].all()
    assert got.outcome[3] == W.ROLLED_BACK
    plain = preempt_walk_ref.walk(snap, bound, pods)
    for k in (0, 1, 2, 4):
        assert (int(got.node[k]), got.victims_of(k)) == (int(plain.node[k]), plain.victims_of(k))
