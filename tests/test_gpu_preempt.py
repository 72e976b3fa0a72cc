"""GPU: bs_preempt and bs_remove_pod bit-exact against the CPU restatement tests/preempt_ref.c (node, n_victims,
n_candidates, offsets, victim lists), the bound-table lifecycle and validation, and round outputs unchanged by it."""
import importlib

import numpy as np
import pytest

import preempt_cases
import preempt_ref
import randsnap

S = importlib.import_module("batch-scheduler_b200.snapshot")
E = importlib.import_module("batch-scheduler_b200.engine")
capi = importlib.import_module("batch-scheduler_b200.capi")

pytestmark = pytest.mark.gpu


def _engine(snap, bound, **kw):
    eng = E.Engine(snap.lanes, **kw)
    eng.upload(snap)
    if bound is not None:
        eng.upload_bound_pods(bound)
    return eng


def _same(got, want):
    np.testing.assert_array_equal(got.node, want.node)
    np.testing.assert_array_equal(got.n_victims, want.n_victims)
    np.testing.assert_array_equal(got.n_candidates, want.n_candidates)
    np.testing.assert_array_equal(got.victim_offset, want.victim_offset)
    np.testing.assert_array_equal(got.victims, want.victims)


def _run(snap, bound, pods=None):
    pods = np.arange(snap.pods.n, dtype=np.uint32) if pods is None else np.asarray(pods, np.uint32)
    eng = _engine(snap, bound)
    got = eng.preempt(pods)
    _same(got, preempt_ref.preempt(snap, bound, pods))
    return eng, got


@pytest.mark.parametrize("name", sorted(preempt_cases.cases()))
def test_hand_built_case(name):
    snap, bound, pods, want = preempt_cases.cases()[name]
    _, got = _run(snap, bound, pods)
    assert [(int(got.node[k]), got.victims_of(k)) for k in range(len(pods))] == want


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("L", [4, 5, 9, 16])
@pytest.mark.parametrize("scale", ["normal", "big"])
def test_random(seed, L, scale):
    snap = randsnap.random_snapshot(seed, P=64, N=90, G=10, L=L, value_scale=scale, aff=4 if seed % 2 else 0)
    bound = S.bound_pods(snap, seed, max_per_node=40, priorities=(-5, 0, 1, 100, 2**31 - 1, -2**31),
                         online=0.3 if seed % 3 else 0.0, locked=0.2 if seed % 4 else 0.0)
    _run(snap, bound)


def test_random_outcomes_are_not_trivial():
    """The random snapshots above reach nodes with victims, not only "no candidate"."""
    chosen = 0
    for seed in range(6):
        snap = randsnap.random_snapshot(seed, P=64, N=90, G=10, L=5, aff=4 if seed % 2 else 0)
        bound = S.bound_pods(snap, seed, max_per_node=40, priorities=(-5, 0, 1, 100, 2**31 - 1, -2**31),
                             online=0.3 if seed % 3 else 0.0, locked=0.2 if seed % 4 else 0.0)
        _, got = _run(snap, bound)
        chosen += int(((got.node >= 0) & (got.n_victims > 0)).sum())
    assert chosen > 0


@pytest.mark.parametrize("seed,N", [(0, 1300), (1, 2049)])
def test_many_node_tiles(seed, N):
    """Several 256-node tiles and a partial last one: the per-tile keys, their reduction in node order."""
    snap = randsnap.random_snapshot(seed, P=48, N=N, G=8, L=5)
    snap.nodes.requested[:3] = snap.nodes.alloc[:3]   # full nodes: a pod fits only where it evicts
    snap.pods.priority[:] = 2**31 - 1
    snap.pods.gid[::2] = S.GID_NONE
    bound = S.bound_pods(snap, seed, max_per_node=12, online=0.5, locked=0.1)
    _, got = _run(snap, bound)
    chosen = got.node[got.node >= 0]
    assert len(got.victims) > 0 and len(set((chosen // 256).tolist())) > 2


def test_ties_across_tiles():
    """Identical nodes in different tiles: the lowest candidate index wins; the nodes of the first two tiles and most
    of the third are unschedulable, so the winner sits in tile 2, and its twins in later tiles tie with it."""
    snap = randsnap.random_snapshot(3, P=16, N=1100, G=4, L=5)
    nt = snap.nodes
    for f in nt.__dataclass_fields__:
        a = getattr(nt, f)
        a[...] = a[..., :1]
    nt.flags[:] = 0
    nt.flags[:700] = S.NODE_UNSCHEDULABLE
    nt.label_mask[:] = ~np.uint64(0)
    nt.taint_mask[:] = 0
    nt.pod_count[:] = 3
    nt.requested[3] = 0
    nt.alloc[3] = 3
    snap.aff_bits = None
    snap.pods.aff_class = None
    snap.pods.gid[:] = S.GID_NONE
    snap.pods.priority[:] = 1000
    snap.pods.req[:] = 0
    snap.pods.req[3] = 1
    snap.pods.req_present[:] = 0
    bound = S.bound_pods(snap, 3, priorities=(5,), n_starts=1, online=1.0)
    _, got = _run(snap, bound)
    assert (got.node == 700).all() and (got.n_candidates == 400).all()


def test_heavy_ties():
    snap = randsnap.random_snapshot(11, P=64, N=70, G=4, L=6)
    bound = S.bound_pods(snap, 11, max_per_node=60, priorities=(0, 1), n_starts=1, online=1.0)
    snap.pods.priority[:] = 5
    snap.pods.gid[:] = S.GID_NONE
    _, got = _run(snap, bound)
    assert (got.n_victims > 1).any()


def test_segment_sizes():
    """Nodes with 0, 1, 33 and more than 1024 bound pods."""
    snap = randsnap.random_snapshot(4, P=40, N=8, G=4, L=5)
    nt = snap.nodes
    nt.flags[:] = 0
    nt.pod_count[:] = [0, 1, 33, 1500, 0, 1, 33, 1500]
    nt.requested[3] = 0
    nt.alloc[3] = 2000
    bound = S.bound_pods(snap, 4, priorities=(-3, 0, 7), n_starts=4, online=1.0)
    np.testing.assert_array_equal(np.bincount(bound.node, minlength=8), nt.pod_count)
    snap.pods.gid[:] = S.GID_NONE
    _run(snap, bound)


def test_many_preemptors():
    snap = randsnap.random_snapshot(7, P=70000, N=40, G=8, L=5)
    bound = S.bound_pods(snap, 7, max_per_node=20)
    pods = np.arange(snap.pods.n, dtype=np.uint32)
    eng = _engine(snap, bound)
    got = eng.preempt(pods)
    sample = np.concatenate([pods[:300], pods[65400:65700], pods[-300:]])
    want = preempt_ref.preempt(snap, bound, sample)
    np.testing.assert_array_equal(got.node[sample], want.node)
    np.testing.assert_array_equal(got.n_victims[sample], want.n_victims)
    np.testing.assert_array_equal(got.n_candidates[sample], want.n_candidates)
    for k, p in enumerate(sample):
        assert got.victims_of(int(p)) == want.victims_of(k)


def test_empty_inputs():
    snap = randsnap.random_snapshot(2, P=20, N=30, G=4, L=5)
    eng, got = _run(snap, S.BoundPodTable.empty(0, 5))
    assert (got.n_victims == 0).all()
    r = eng.preempt(np.zeros(0, np.uint32))
    assert len(r.node) == 0 and list(r.victim_offset) == [0]
    empty = randsnap.random_snapshot(2, P=20, N=0, G=4, L=5)
    eng2, got2 = _run(empty, S.BoundPodTable.empty(0, 5))
    assert (got2.node == -1).all() and (got2.n_candidates == 0).all()


def test_remove_pod_codes():
    snap = randsnap.random_snapshot(1, P=3, N=4, G=3, L=4)
    snap.pods.gid[:] = [S.GID_NONE, S.GID_MISSING, 0]
    rows = [(S.GID_NONE, 0), (S.GID_MISSING, 0), (0, 0), (0, 1), (1, 0), (1, 1)]
    bound = S.BoundPodTable.empty(len(rows), 4)
    bound.node[:] = 0
    snap.nodes.pod_count[0] = len(rows)
    bound.gid[:] = [g for g, _ in rows]
    bound.flags[:] = [f for _, f in rows]
    eng = _engine(snap, bound)
    seen = set()
    for p in range(3):
        for v in range(len(rows)):
            code, reason, group = eng.remove_pod(p, v)
            want = preempt_ref.remove_pod(int(snap.pods.gid[p]), rows[v][0], rows[v][1])
            assert reason == want
            assert code == (capi.CODE_SUCCESS if want == capi.REMOVE_ALLOW else capi.CODE_UNSCHEDULABLE)
            assert group == (rows[v][0] if rows[v][0] >= 0 else -1)
            seen.add(reason)
    assert seen == set(range(5))


def _bound_for(snap, seed=0):
    return S.bound_pods(snap, seed, max_per_node=10)


def test_lifecycle_drops_table():
    snap = randsnap.random_snapshot(3, P=10, N=20, G=4, L=5)
    bound = _bound_for(snap)
    pods = np.arange(10, dtype=np.uint32)
    for drop in ("nodes", "update", "groups"):
        eng = _engine(snap, bound)
        eng.preempt(pods)
        if drop == "nodes":
            eng.upload_nodes(snap.nodes)
        elif drop == "update":
            eng.update_nodes([0], S.NodeTable(*(getattr(snap.nodes, f)[..., :1] for f in snap.nodes.__dataclass_fields__)))
        else:
            eng.upload_groups(snap.groups)
        with pytest.raises(capi.BsError) as ex:
            eng.preempt(pods)
        assert ex.value.code == capi.BS_E_STATE
        with pytest.raises(capi.BsError) as ex:
            eng.remove_pod(0, 0)
        assert ex.value.code == capi.BS_E_STATE


def test_validation_errors():
    snap = randsnap.random_snapshot(3, P=10, N=20, G=4, L=5)
    good = _bound_for(snap)
    eng = _engine(snap, good)
    pods = np.arange(10, dtype=np.uint32)
    ref = eng.preempt(pods)

    def expect(bt, code):
        with pytest.raises(capi.BsError) as ex:
            eng.upload_bound_pods(bt)
        assert ex.value.code == code
        with pytest.raises(capi.BsError) as ex2:   # the failing table is dropped
            eng.preempt(pods)
        assert ex2.value.code == capi.BS_E_STATE
        eng.upload_bound_pods(good)
        _same(eng.preempt(pods), ref)

    bt = good.copy(); bt.node[0] = snap.nodes.n
    expect(bt, capi.BS_E_INDEX)
    n0 = int(good.node[0])
    extra = int(snap.nodes.pod_count[n0]) - int((good.node == n0).sum()) + 1
    bt = S.BoundPodTable(*(np.concatenate([getattr(good, f), np.repeat(getattr(good, f)[..., :1], extra, axis=-1)], axis=-1)
                           for f in good.__dataclass_fields__))
    expect(bt, capi.BS_E_INVAL)
    lacks = np.nonzero((snap.nodes.req_present[good.node] & np.uint32(1 << 4)) == 0)[0]
    assert len(lacks), "some row sits on a node without scalar key 4"
    bt = good.copy(); bt.req_present[lacks[0]] |= np.uint32(1 << 4)
    expect(bt, capi.BS_E_INVAL)
    bt = good.copy(); bt.gid[0] = -3   # neither a group, online nor missing
    expect(bt, capi.BS_E_INDEX)
    bt = good.copy(); bt.req[0, 0] = (1 << 56) + 1
    expect(bt, capi.BS_E_RANGE)
    n2 = int(np.nonzero(np.bincount(good.node, minlength=snap.nodes.n) >= 2)[0][0])
    v = np.nonzero(good.node == n2)[0][:2]
    bt = good.copy(); bt.req[1, v] = 1 << 56   # each value in range, their sum is not
    expect(bt, capi.BS_E_RANGE)
    bt = good.copy(); bt.req[3, 0] = 1 << 60   # lane 3 is ignored
    eng.upload_bound_pods(bt)
    _same(eng.preempt(pods), ref)
    bt = good.copy(); bt.req[1, 0] = -(1 << 56) - 1
    expect(bt, capi.BS_E_RANGE)
    bt = good.copy(); bt.gid[0] = snap.groups.n
    eng.upload_bound_pods(bt)
    with pytest.raises(capi.BsError) as ex:
        eng.preempt(pods)
    assert ex.value.code == capi.BS_E_INDEX


def test_victims_cap_too_small():
    snap = randsnap.random_snapshot(5, P=30, N=30, G=4, L=5)
    bound = S.bound_pods(snap, 5, max_per_node=20, online=1.0)
    snap.pods.gid[:] = S.GID_NONE
    snap.pods.priority[:] = 2**31 - 1
    eng = _engine(snap, bound)
    full = eng.preempt(np.arange(30, dtype=np.uint32))
    assert len(full.victims) > 0
    r = capi.PreemptResultC()
    n = 30
    idx = np.arange(n, dtype=np.uint32)
    node, nv, cand, off = np.zeros(n, np.int32), np.zeros(n, np.uint32), np.zeros(n, np.uint32), np.zeros(n + 1, np.uint32)
    vict = np.full(4, 7, np.uint32)
    r = capi.PreemptResultC(capi.ptr(node), capi.ptr(nv), capi.ptr(cand), capi.ptr(off), capi.ptr(vict),
                            len(full.victims) - 1, 0)
    import ctypes as C
    rc = eng.lib.bs_preempt(eng.h, capi.ptr(idx), n, C.byref(r))
    assert rc == capi.BS_E_INVAL and r.victims_total == len(full.victims)
    assert (vict == 7).all()


def test_independent_of_rounds():
    """The same answer with and without a prior round, and round outputs byte-identical with a bound table."""
    snap = randsnap.random_snapshot(9, P=80, N=100, G=10, L=6, aff=3)
    bound = S.bound_pods(snap, 9, max_per_node=30)
    pods = np.arange(snap.pods.n, dtype=np.uint32)
    base = E.Engine(snap.lanes, fit_bitmap=True, reasons=True)
    base.upload(snap)
    r0 = base.evaluate()
    fit0, reasons0 = base.fit_rows(), base.reason_rows()
    a = _engine(snap, bound, fit_bitmap=True, reasons=True)
    first = a.preempt(pods)
    r1 = a.evaluate()
    second = a.preempt(pods)
    _same(first, second)
    _same(first, preempt_ref.preempt(snap, bound, pods))
    for f in r0.__dataclass_fields__:
        x, y = getattr(r0, f), getattr(r1, f)
        if isinstance(x, np.ndarray):
            assert x.tobytes() == y.tobytes(), f
        else:
            assert x == y, f
    assert fit0.tobytes() == a.fit_rows().tobytes()
    assert reasons0.tobytes() == a.reason_rows().tobytes()
    b = _engine(snap, None, fit_bitmap=True, reasons=True)
    b.evaluate()
    b.upload_bound_pods(bound)
    _same(b.preempt(pods), first)
