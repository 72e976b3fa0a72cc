"""GPU: bs_replay_priority — the pod-at-a-time walk with kube-scheduler's node choice — bit-exact against the CPU
restatement tests/replay_priority_ref.c per queue position and on the whole after-state including the live non-zero
column, in every lane build, for several weight sets, with the cross-layer and error checks of the C ABI and full-size
properties at cfg4."""
import json
import subprocess

import numpy as np
import pytest

import native
import priority_ref
import pyref_priority
import replay_priority_ref as rpr
from randsnap import S, random_snapshot

pytestmark = pytest.mark.gpu

WEIGHTS = [(1, 0, 1), (0, 1, 0), (1, 1, 1), (3, 0, 7)]
AFTER = ("node_requested", "node_pod_count", "node_req_present", "group_matched", "group_flags", "group_min_res",
         "group_min_res_present", "group_rep_sel", "group_rep_tol")


def _engine(pkg, snap, node_nz, pod_nz, weights):
    eng = pkg.Engine(snap.lanes)
    eng.upload(snap)
    eng.upload_nonzero(node=node_nz, pods=pod_nz)
    eng.set_score_weights(*weights)
    return eng


def walk_both(pkg, snap, queue=None, weights=(1, 0, 1), nz=None, seed=0):
    node_nz, pod_nz = S.nonzero_requests(snap, seed) if nz is None else nz
    eng = _engine(pkg, snap, node_nz, pod_nz, weights)
    try:
        got = eng.replay(queue, priority=True)
        # the uploaded tables and columns are untouched: a second walk gives the same answer
        again = eng.replay(queue, after_state=False, priority=True)
    finally:
        eng.close()
    pf, node, ready, after, nz_after = rpr.replay_priority(snap, node_nz, pod_nz, queue, weights)
    np.testing.assert_array_equal(got["prefilter"], pf)
    np.testing.assert_array_equal(got["node"], node)
    np.testing.assert_array_equal(got["ready"], ready)
    for k in ("prefilter", "node", "ready"):
        np.testing.assert_array_equal(again[k], got[k])
    nt, gt = after.nodes, after.groups
    want = dict(node_requested=nt.requested, node_pod_count=nt.pod_count, node_req_present=nt.req_present,
                group_matched=gt.matched, group_flags=gt.flags, group_min_res=gt.min_res,
                group_min_res_present=gt.min_res_present, group_rep_sel=gt.rep_sel, group_rep_tol=gt.rep_tol)
    for k in AFTER:
        np.testing.assert_array_equal(got[k], want[k], err_msg=k)
    np.testing.assert_array_equal(got["node_nonzero"], nz_after)
    return got


@pytest.mark.parametrize("seed", range(20))
def test_random_snapshots(pkg, oracle, seed):
    case = ["mixed", "A", "B"][seed % 3]
    L = [6, 4, 5, 9, 12, 16][seed % 6]   # MAXL 9, 5, 5, 9, 16, 16
    N = [70, 1500, 2600, 5000][seed % 4]
    snap = random_snapshot(1000 + seed, P=300, N=N, G=40, L=L, case=case)
    queue = None if seed % 2 == 0 else np.random.default_rng(seed).permutation(snap.pods.n)
    walk_both(pkg, snap, queue, WEIGHTS[seed % 4], seed=seed)


@pytest.mark.parametrize("L", [5, 9, 16])
@pytest.mark.parametrize("w", WEIGHTS)
def test_lane_builds_and_weights(pkg, oracle, L, w):
    snap = random_snapshot(1100 + L, P=260, N=1500, G=30, L=L, case="mixed")
    walk_both(pkg, snap, None, w, seed=L)


@pytest.mark.parametrize("seed", range(4))
def test_affinity_classes(pkg, oracle, seed):
    snap = random_snapshot(300 + seed, P=260, N=90 + 300 * seed, G=14, L=[5, 6][seed % 2], aff=2 + seed)
    walk_both(pkg, snap, None, WEIGHTS[seed], seed=seed)


def test_more_classes_than_the_block_cache_holds(pkg, oracle):
    snap = random_snapshot(91, P=300, N=2600, G=40, L=5, case="mixed")
    rng = np.random.default_rng(91)
    snap.pods.tol_mask[:] = rng.integers(0, 1 << 20, snap.pods.n).astype(np.uint64) | np.uint64(0xF)
    walk_both(pkg, snap, None, (1, 1, 1), seed=91)


@pytest.mark.parametrize("w", WEIGHTS)
def test_identical_nodes(pkg, oracle, w):
    """Tie-heavy: every node the same, so every choice is decided by the live columns and the index."""
    snap = random_snapshot(17, P=300, N=2100, G=30, L=5)
    nt = snap.nodes
    nt.flags[:] = 0
    nt.label_mask[:] = 0xF
    nt.taint_mask[:] = 0
    nt.alloc[0], nt.alloc[1], nt.alloc[2], nt.alloc[3] = 8000, 1 << 34, 1 << 36, 110
    nt.requested[:] = 0
    nt.pod_count[:] = 0
    node_nz = np.zeros((2, nt.n), np.int64)
    pod_nz = np.stack([snap.pods.req[0].clip(0, None), snap.pods.req[1].clip(0, None)]).astype(np.int64)
    got = walk_both(pkg, snap, None, w, nz=(node_nz, pod_nz))
    assert (got["node"] >= 0).any()


def test_binary64_balanced(pkg, oracle):
    """cpu 10/1000 against memory 560/1000 gives Balanced 44 in binary64 (45 in exact arithmetic), 559/1000 gives 45:
    the pod goes to node 1, where exact arithmetic would tie and pick node 0."""
    assert pyref_priority.score(10, 1000, 560, 1000, (0, 0, 1)) == 44
    assert pyref_priority.score(10, 1000, 559, 1000, (0, 0, 1)) == 45
    L = 4
    nt = S.NodeTable.empty(2, L)
    nt.alloc[0], nt.alloc[1], nt.alloc[3] = 1000, 1000, 110
    pt = S.PodTable.empty(1, L)
    pt.req[0], pt.req[1] = 10, 559
    snap = S.Snapshot(nt, pt, S.GroupTable.empty(0, L), "binary64")
    nz = (np.array([[0, 0], [1, 0]], np.int64), np.array([[10], [559]], np.int64))
    got = walk_both(pkg, snap, None, (0, 0, 1), nz=nz)
    assert got["node"].tolist() == [1] and got["node_nonzero"].tolist() == [[0, 10], [1, 559]]


def test_negative_allocatable_and_requests(pkg, oracle):
    snap = random_snapshot(451, P=300, N=1200, G=20, L=5)
    nt, pt = snap.nodes, snap.pods
    rng = np.random.default_rng(451)
    neg = rng.random(nt.n) < 0.3
    nt.alloc[1, neg] = -(1 << 20)
    nt.requested[1, neg] = -(1 << 30)
    pt.req[1] = np.where(rng.random(pt.n) < 0.3, -(1 << 10), pt.req[1])
    for w in WEIGHTS:
        walk_both(pkg, snap, None, w, seed=451)


def test_no_nodes(pkg, oracle):
    snap = random_snapshot(5, P=50, N=1, G=8, L=5, case="mixed")
    snap.nodes = snap.nodes.take(np.zeros(0, np.int64))
    nz = (np.zeros((2, 0), np.int64), S.nonzero_requests(snap, 5)[1])
    got = walk_both(pkg, snap, None, (1, 0, 1), nz=nz)
    assert (got["node"] == -1).all() and got["node_nonzero"].shape == (2, 0)


def test_repeated_and_empty_queue(pkg, oracle):
    snap = random_snapshot(5, P=50, N=40, G=8, L=5, case="mixed")
    walk_both(pkg, snap, np.array([3, 3, 7, 3, 0, 49, 49], np.uint32), seed=5)
    walk_both(pkg, snap, np.zeros(0, np.uint32), seed=5)


def test_cfg4_third_scale_device_order(pkg, oracle, snapshot_mod):
    snap = snapshot_mod.config(4, scale=0.3)
    eng = pkg.Engine(snap.lanes, fit_bitmap=False, score=False)
    eng.upload(snap)
    order = eng.evaluate().order.copy()
    eng.close()
    got = walk_both(pkg, snap, order, (1, 0, 1), seed=4)
    assert got["ready"].sum() > 1000


@pytest.mark.parametrize("w", WEIGHTS)
def test_first_pass_is_the_round_priority_entry(pkg, oracle, w):
    """Before the first assume the live state is the uploaded one: the first passing pod's node is entry 0 of its
    K = 1 BS_OUT_PRIORITY list on the same tables."""
    snap = random_snapshot(23, P=300, N=1500, G=30, L=6, case="mixed")
    node_nz, pod_nz = S.nonzero_requests(snap, 23)
    queue = np.random.default_rng(23).permutation(snap.pods.n)
    eng = _engine(pkg, snap, node_nz, pod_nz, w)
    try:
        got = eng.replay(queue, priority=True)
    finally:
        eng.close()
    first = int(np.flatnonzero(got["prefilter"] == S.PF_PASS)[0])
    eng = pkg.Engine(snap.lanes, 0, priority_k=1)
    try:
        eng.upload(snap)
        eng.upload_nonzero(node=node_nz, pods=pod_nz)
        eng.set_score_weights(*w)
        eng.evaluate()
        nodes, _ = eng.priority_rows()
    finally:
        eng.close()
    assert got["node"][first] == nodes[queue[first], 0]
    np.testing.assert_array_equal(nodes[:, 0], priority_ref.priority_rows(snap, node_nz, pod_nz, 1, w)[0][:, 0])


@pytest.mark.parametrize("seed", range(3))
def test_zero_weights_are_bs_replay(pkg, oracle, seed):
    snap = random_snapshot(40 + seed, P=300, N=[70, 2600, 5000][seed], G=40, L=[5, 9, 16][seed], aff=2 * seed)
    node_nz, pod_nz = S.nonzero_requests(snap, seed)
    eng = _engine(pkg, snap, node_nz, pod_nz, (0, 0, 0))
    try:
        scored = eng.replay(None, priority=True)
        first = eng.replay(None)
    finally:
        eng.close()
    for k, v in first.items():
        np.testing.assert_array_equal(scored[k], v, err_msg=k)


def test_errors(pkg):
    c = pkg.capi
    snap = random_snapshot(601, P=50, N=80, G=5, L=6)
    node_nz, pod_nz = S.nonzero_requests(snap, 601)

    def code(f, *a, **kw):
        with pytest.raises(c.BsError) as ei:
            f(*a, **kw)
        return ei.value.code

    eng = pkg.Engine(snap.lanes)
    try:
        eng.upload(snap)
        assert code(eng.replay, priority=True) == c.BS_E_STATE            # no columns
        eng.upload_nonzero(node=node_nz)
        assert code(eng.replay, priority=True) == c.BS_E_STATE            # no pod column
        eng.upload_nonzero(pods=pod_nz)
        eng.replay(priority=True)
        eng.update_nodes(np.array([3]), snap.nodes.take([3]))
        assert code(eng.replay, priority=True) == c.BS_E_STATE            # row updates drop the node column
        eng.upload_nonzero(node=node_nz)
        eng.replay(priority=True)
        eng.upload_nodes(snap.nodes)
        assert code(eng.replay, priority=True) == c.BS_E_STATE            # so does a node upload
        eng.replay()                                                      # bs_replay needs no column
        # the live sums: max(node) + n_queue * max(pod) must stay within 2^62
        big = np.full((2, snap.pods.n), c.NONZERO_MAX, np.int64)
        eng.upload_nonzero(node=np.full((2, snap.nodes.n), c.NONZERO_MAX, np.int64), pods=big)
        eng.replay(np.arange(63, dtype=np.uint32) % snap.pods.n, priority=True)   # 64 * 2^56 = 2^62
        assert code(eng.replay, np.arange(64, dtype=np.uint32) % snap.pods.n, priority=True) == c.BS_E_RANGE
    finally:
        eng.close()


def test_full_size_cfg4(pkg, snapshot_mod):
    """100k pods in device order, checked by properties: (0, 0, 0) is bs_replay; under (1, 0, 1) the live column and
    `requested` grow by exactly the assumed pods' columns and requests."""
    snap = snapshot_mod.config(4)
    node_nz, pod_nz = snapshot_mod.nonzero_requests(snap, 4)
    eng = pkg.Engine(snap.lanes, fit_bitmap=False, score=False)
    try:
        eng.upload(snap)
        order = eng.evaluate().order.copy()
        eng.upload_nonzero(node=node_nz, pods=pod_nz)
        first = eng.replay(order)
        eng.set_score_weights(0, 0, 0)
        zero = eng.replay(order, priority=True)
        eng.set_score_weights(1, 0, 1)
        got = eng.replay(order, priority=True)
    finally:
        eng.close()
    for k, v in first.items():
        np.testing.assert_array_equal(zero[k], v, err_msg=k)
    placed = got["node"] >= 0
    assert placed.sum() > 1000 and (got["node"] != first["node"]).any()
    pods = order[placed]
    want = node_nz.copy()
    req = snap.nodes.requested.copy()
    for r in range(2):
        np.add.at(want[r], got["node"][placed], pod_nz[r, pods])
        np.add.at(req[r], got["node"][placed], snap.pods.req[r, pods])
    np.testing.assert_array_equal(got["node_nonzero"], want)
    np.testing.assert_array_equal(got["node_requested"][:2], req[:2])
    np.testing.assert_array_equal(np.bincount(got["node"][placed], minlength=snap.nodes.n),
                                  got["node_pod_count"] - snap.nodes.pod_count)


def test_plugin_replay_queue_choices():
    """BatchSchedulingPlugin::ReplayQueue: two empty 4-cpu / 8Gi nodes, four 500m / 1Gi pods.  First-fit packs node 0;
    kPriority under (1, 0, 1) alternates (87 + 100 on both empty nodes, then 175 against 187, ...), under (0, 1, 0)
    packs node 0; without priority_k kPriority is an error."""
    o = json.loads(subprocess.check_output([native.cpp_program("plugin_replay_priority_test")], text=True))
    assert o["first_fit"] == o["plain_first_fit"] == [0, 0, 0, 0]
    assert o["least_balanced"] == [0, 1, 0, 1] and o["positions"] == [0, 1, 2, 3]
    assert o["most"] == [0, 0, 0, 0]
    assert o["no_priority_k_fails"] == 1 and "priority_k" in o["message"]
