"""GPU: bs_preempt_walk bit-exact against the CPU restatement tests/preempt_walk_ref.c (node, n_victims, n_candidates,
offsets, victims in order, outcome, evicted_by): the hand-built cases of tests/preempt_walk_cases.py, random tables at
every register width of the kernels (MAXL 5, 9 and 16) with and without gang units and PodDisruptionBudget bits,
several node tiles with ties across them, N = 0 and n = 0, a victims cap that is too small, every refusal, two walks
giving one answer, and bs_preempt's answers unchanged by a walk."""
import ctypes as C
import importlib
import itertools

import numpy as np
import pytest

import preempt_walk_cases as W
import preempt_walk_ref
import randsnap

S = importlib.import_module("batch-scheduler_b200.snapshot")
E = importlib.import_module("batch-scheduler_b200.engine")
capi = importlib.import_module("batch-scheduler_b200.capi")

pytestmark = pytest.mark.gpu


def _engine(snap, bound):
    eng = E.Engine(snap.lanes)
    eng.upload(snap)
    eng.upload_bound_pods(bound)
    return eng


def _same(got, want):
    np.testing.assert_array_equal(got.node, want.node)
    np.testing.assert_array_equal(got.n_victims, want.n_victims)
    np.testing.assert_array_equal(got.n_candidates, want.n_candidates)
    np.testing.assert_array_equal(got.victim_offset, want.victim_offset)
    np.testing.assert_array_equal(got.victims, want.victims)
    np.testing.assert_array_equal(got.outcome, want.outcome)
    np.testing.assert_array_equal(got.evicted_by, want.evicted_by)


def _run(snap, bound, pods, gang=False):
    eng = _engine(snap, bound)
    got = eng.preempt_walk(np.asarray(pods, np.uint32), gang=gang)
    eng.close()
    _same(got, preempt_walk_ref.walk(snap, bound, pods, gang))
    return got


@pytest.mark.parametrize("name", sorted(W.cases()))
def test_hand_built_case(name):
    snap, bound, pods, gang, want, _ = W.cases()[name]
    got = _run(snap, bound, pods, gang)
    assert [(int(got.node[k]), got.victims_of(k), int(got.outcome[k])) for k in range(len(pods))] == want


@pytest.mark.parametrize("seed,L,violating,gang",
                         list(itertools.product((0, 2, 4), (5, 9, 16), (0.0, 0.5), (False, True))))
def test_random(seed, L, violating, gang):
    """L 5, 9 and 16 run the MAXL 5, 9 and 16 builds of the node and commit kernels."""
    snap, bound = W.random_table(seed, L, violating, P=64, N=90, G=10, max_per_node=40)
    pods = W.queue(snap, gang=gang)
    got = _run(snap, bound, pods, gang)
    assert len(got.victims) > 0
    assert not gang or (got.outcome == W.ROLLED_BACK).any()


def test_many_node_tiles():
    """Several 256-node tiles and a partial last one, full nodes, 200 online preemptors competing for them."""
    snap = randsnap.random_snapshot(1, P=200, N=1300, G=8, L=5)
    snap.nodes.requested[:3] = snap.nodes.alloc[:3]
    snap.pods.priority[:] = 2**31 - 1
    snap.pods.gid[:] = S.GID_NONE
    bound = S.bound_pods(snap, 1, max_per_node=12, online=0.5, locked=0.1, violating=0.3)
    got = _run(snap, bound, list(range(200)))
    chosen = got.node[got.node >= 0]
    assert len(got.victims) > 0 and len(set((chosen // 256).tolist())) > 2


def test_ties_across_tiles():
    """Identical nodes 700-1099 in three tiles, one pod slot each held by a prio-5 bound pod.  Each preemptor takes the
    lowest-indexed node left, across the tile borders at 768 and 1024."""
    snap = randsnap.random_snapshot(3, P=400, N=1100, G=4, L=5)
    nt = snap.nodes
    for f in nt.__dataclass_fields__:
        a = getattr(nt, f)
        a[...] = a[..., :1]
    nt.flags[:] = 0
    nt.flags[:700] = S.NODE_UNSCHEDULABLE
    nt.label_mask[:] = ~np.uint64(0)
    nt.taint_mask[:] = 0
    nt.pod_count[:] = 1
    nt.requested[3] = 0
    nt.alloc[3] = 1
    snap.aff_bits = None
    snap.pods.aff_class = None
    snap.pods.gid[:] = S.GID_NONE
    snap.pods.priority[:] = 1000
    snap.pods.req[:] = 0
    snap.pods.req[3] = 1
    snap.pods.req_present[:] = 0
    bound = S.bound_pods(snap, 3, priorities=(5,), n_starts=1, online=1.0)
    got = _run(snap, bound, list(range(400)))
    assert got.node.tolist() == list(range(700, 1100))
    assert got.n_candidates.tolist() == list(range(400, 0, -1))


def test_no_nodes_and_no_preemptors():
    snap, _ = W.random_table(4, 5, 0.0)
    snap.nodes = S.NodeTable.empty(0, 5)
    snap.aff_bits = None
    snap.pods.aff_class = None
    snap.pods.gid[:] = S.GID_NONE
    bound = S.BoundPodTable.empty(0, 5)
    pods = W.queue(snap)
    for gang in (False, True):
        got = _run(snap, bound, pods, gang)
        assert (got.node == -1).all() and (got.n_candidates == 0).all()
        assert (got.outcome == (W.ROLLED_BACK if gang else W.NONE)).all()
    snap, bound = W.random_table(4, 5, 0.5)
    got = _run(snap, bound, [])
    assert len(got.node) == 0 and (got.evicted_by == -1).all() and got.victim_offset.tolist() == [0]


def _walk_c(eng, pods, flags=0, cap=1 << 20):
    idx = np.asarray(pods, np.uint32)
    n = len(idx)
    node, nv, cand, off = np.zeros(n, np.int32), np.zeros(n, np.uint32), np.zeros(n, np.uint32), np.zeros(n + 1, np.uint32)
    vict = np.full(max(cap, 1), 7, np.uint32)
    r = capi.PreemptResultC(capi.ptr(node), capi.ptr(nv), capi.ptr(cand), capi.ptr(off), capi.ptr(vict), cap, 0)
    rc = eng.lib.bs_preempt_walk(eng.h, capi.ptr(idx) if n else None, n, flags, C.byref(r), None, None)
    return rc, r, vict


def test_victims_cap_too_small():
    snap, bound = W.random_table(5, 5, 0.5, P=30, N=30)
    snap.pods.gid[:] = S.GID_NONE
    snap.pods.priority[:] = 2**31 - 1
    eng = _engine(snap, bound)
    pods = list(range(30))
    full = eng.preempt_walk(pods)
    _same(full, preempt_walk_ref.walk(snap, bound, pods))
    assert len(full.victims) > 0
    rc, r, vict = _walk_c(eng, pods, cap=len(full.victims) - 1)
    eng.close()
    assert rc == capi.BS_E_INVAL and r.victims_total == len(full.victims)
    assert (vict == 7).all()


def test_refusals():
    snap, bound = W.random_table(6, 5, 0.0, P=10, G=3)
    pt = snap.pods
    pt.priority[:] = 10
    pt.priority[1] = 20
    pt.gid[:] = S.GID_NONE
    pt.gid[[2, 3, 5]] = 1
    eng = _engine(snap, bound)
    assert _walk_c(eng, [0, 1])[0] == capi.BS_E_INVAL            # priority rises along the list
    assert _walk_c(eng, [1, 0, 0])[0] == capi.BS_E_INVAL         # a pod listed twice
    assert _walk_c(eng, [1, 0], flags=2)[0] == capi.BS_E_INVAL   # an unknown flag bit
    assert _walk_c(eng, [2, 4, 3], flags=capi.PREEMPT_GANG)[0] == capi.BS_E_INVAL   # group 1 split
    assert _walk_c(eng, [2, 4, 3])[0] == capi.BS_OK               # without gang units the split is allowed
    assert _walk_c(eng, [2, 3, 5, 4], flags=capi.PREEMPT_GANG)[0] == capi.BS_OK
    assert _walk_c(eng, [1, 99])[0] == capi.BS_E_INDEX
    eng.close()
    eng = E.Engine(snap.lanes)
    eng.upload(snap)
    assert _walk_c(eng, [0])[0] == capi.BS_E_STATE               # no bound-pod table
    eng.close()


def test_live_sums_range():
    snap, bound = W.random_table(7, 5, 0.0, P=300, N=8)
    snap.pods.req[0] = -(1 << 56)
    snap.pods.gid[:] = S.GID_NONE
    snap.pods.priority[:] = 5
    eng = _engine(snap, bound)
    assert _walk_c(eng, list(range(300)))[0] == capi.BS_E_RANGE   # 300 nominations of -2^56 pass 2^62
    assert _walk_c(eng, list(range(10)))[0] == capi.BS_OK
    eng.close()


def test_deterministic_and_state_unchanged():
    snap, bound = W.random_table(8, 9, 0.5, P=64, N=90, G=10, max_per_node=40)
    pods = W.queue(snap, gang=True)
    eng = _engine(snap, bound)
    before = eng.preempt(pods)
    a = eng.preempt_walk(pods, gang=True)
    b = eng.preempt_walk(pods, gang=True)
    after = eng.preempt(pods)
    eng.close()
    _same(a, b)
    for f in ("node", "n_victims", "n_candidates", "victim_offset", "victims"):
        np.testing.assert_array_equal(getattr(before, f), getattr(after, f))
    assert len(a.victims) > 0


def test_gid_past_the_group_table_is_a_unit_of_one():
    """A pod whose gid is >= n_groups names no group of the table: under gang units it is a unit of one, as a
    missing group is.  Four such pods share one gid, two of them side by side, and the one that fits nowhere rolls
    back alone; the group-1 pair in between is one unit."""
    snap, bound = W.random_table(9, 5, 0.5, P=12, N=8, G=3)
    pt = snap.pods
    pt.priority[:] = 2**31 - 1
    pt.gid[:] = S.GID_NONE
    pt.gid[[0, 2, 5, 6]] = snap.groups.n + 4
    pt.gid[[3, 4]] = 1
    pt.req[0, 2] = 1 << 50
    pods = list(range(12))
    got = _run(snap, bound, pods, gang=True)
    plain = _run(snap, bound, pods, gang=False)
    assert got.outcome[2] == W.ROLLED_BACK and plain.outcome[2] == W.NONE
    for k in (0, 1, 5, 6):
        assert (int(got.node[k]), got.victims_of(k)) == (int(plain.node[k]), plain.victims_of(k))
    assert len(got.victims) > 0
