"""GPU: the RequestedToCapacityRatio priority (bs_set_ratio_priority) in the round's priority lists and in
bs_replay_priority, bit-exact against the CPU restatement tests/ratio_priority_ref.c: every lane build, unaligned sizes,
list lengths, shapes, weight sets, extreme and negative values; weight 0 is the engine without the priority; every
BS_E_INVAL case keeps the previous setting; and the C++ plugin's SetRatioPriority."""
import json
import os
import subprocess

import numpy as np
import pytest

import priority_ref
import ratio_priority_ref as rr
from randsnap import S, random_snapshot

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPES = {"default": rr.DEFAULT_SHAPE, "binpack": rr.BIN_PACK, "single": ((50, 40),),
          "full": tuple((u, (u * 37) % 101) for u in range(101)), "falling": ((0, 100), (30, 0)),
          "rising": ((10, 20), (40, 90), (60, 30), (100, 70))}
WEIGHTS = [(0, 0, 0), (1, 0, 1), (0, 1, 0)]
AFTER = ("node_requested", "node_pod_count", "node_req_present", "group_matched", "group_flags", "group_min_res",
         "group_min_res_present", "group_rep_sel", "group_rep_tol")


def _sub(table, idx):
    return type(table)(*(None if getattr(table, f) is None else
                         (getattr(table, f)[:, idx] if getattr(table, f).ndim == 2 else getattr(table, f)[idx])
                         for f in table.__dataclass_fields__))


def _lane_weights(L, seed, gpu_only=False):
    if gpu_only:
        return [0, 0, 0, 0, 3] + [0] * (L - 5)
    rng = np.random.default_rng(seed)
    lw = [int(x) for x in rng.integers(0, 4, L)]
    lw[3] = 0
    return lw


def _rows(pkg, snap, K, weights, ratio, nz):
    eng = pkg.Engine(snap.lanes, 0, priority_k=K)
    try:
        eng.upload(snap)
        eng.upload_nonzero(node=nz[0], pods=nz[1])
        eng.set_score_weights(*weights)
        if ratio is not None:
            eng.set_ratio_priority(ratio[0], ratio[1], ratio[2], ratio[3])
        eng.evaluate()
        return eng.priority_rows()
    finally:
        eng.close()


def _check_rows(pkg, snap, K, weights, ratio, seed=0, nz=None):
    nz = S.nonzero_requests(snap, seed) if nz is None else nz
    nodes, scores = _rows(pkg, snap, K, weights, ratio, nz)
    want_n, want_s = rr.priority_rows(snap, nz[0], nz[1], K, ratio, weights)
    np.testing.assert_array_equal(nodes, want_n)
    np.testing.assert_array_equal(scores, want_s)
    return nodes, scores


@pytest.mark.parametrize("L", [5, 9, 16])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_lane_builds_and_shapes(pkg, oracle, L, shape):
    snap = random_snapshot(900 + L, P=260, N=700, G=30, L=L, case="mixed")
    K = {5: 1, 9: 7, 16: 32}[L]
    w = WEIGHTS[len(shape) % 3]
    _check_rows(pkg, snap, K, w, (1 + L % 3, SHAPES[shape], _lane_weights(L, L), L % 2), seed=L)


@pytest.mark.parametrize("w", WEIGHTS)
@pytest.mark.parametrize("K", [1, 7, 32])
def test_weight_sets_and_lengths(pkg, oracle, w, K):
    snap = random_snapshot(950 + K, P=300, N=900, G=30, L=6, aff=3)
    _check_rows(pkg, snap, K, w, (2, rr.BIN_PACK, _lane_weights(6, K), 1), seed=K)


@pytest.mark.parametrize("N", [0, 1, 31, 33, 511, 1025])
def test_unaligned_sizes(pkg, oracle, N):
    snap = random_snapshot(N * 5 + 1, P=70, N=max(N, 1), G=9, L=6)
    if N == 0:
        snap.nodes = _sub(snap.nodes, np.zeros(0, np.int64))
    nodes, _ = _check_rows(pkg, snap, 7, (1, 0, 1), (1, rr.BIN_PACK, [1, 1, 1, 0, 2, 2], 1), seed=N)
    if N == 0:
        assert (nodes == -1).all()


@pytest.mark.parametrize("L", [5, 9, 16])
def test_gpu_lane_only(pkg, oracle, L):
    """cfg4's shape of problem: only lane 4 weighs, nodes with 0 / 4 / 8 of it, pods asking 0-8."""
    snap = random_snapshot(980 + L, P=300, N=800, G=30, L=L, case="mixed")
    nt, pt = snap.nodes, snap.pods
    rng = np.random.default_rng(L)
    gpus = rng.choice([0, 4, 8], nt.n)
    nt.alloc[4] = gpus
    bit = np.uint32(1 << 4)
    nt.alloc_present = np.where(gpus > 0, nt.alloc_present | bit, nt.alloc_present & ~bit).astype(np.uint32)
    nt.requested[4] = np.minimum(gpus, rng.integers(0, 5, nt.n))
    nt.req_present |= bit
    pt.req[4] = rng.integers(0, 9, pt.n)
    pt.req_present = np.where(pt.req[4] > 0, pt.req_present | bit, pt.req_present & ~bit).astype(np.uint32)
    for w in WEIGHTS:
        _check_rows(pkg, snap, 16, w, (1, rr.BIN_PACK, _lane_weights(L, 0, gpu_only=True), 0), seed=L)
        _check_rows(pkg, snap, 16, w, (3, rr.DEFAULT_SHAPE, [1, 1, 0, 0, 3] + [0] * (L - 5), 2), seed=L)


def test_extreme_and_negative_values(pkg, oracle):
    snap = random_snapshot(991, P=300, N=1200, G=20, L=9, value_scale="big")
    nt, pt = snap.nodes, snap.pods
    rng = np.random.default_rng(991)
    lim = 1 << 56
    for d in (2, 4, 5, 6):
        nt.alloc[d] = np.where(rng.random(nt.n) < 0.2, -lim, np.where(rng.random(nt.n) < 0.2, lim, nt.alloc[d]))
        nt.requested[d] = np.where(rng.random(nt.n) < 0.2, -lim, np.where(rng.random(nt.n) < 0.1, lim, nt.requested[d]))
        pt.req[d] = np.where(rng.random(pt.n) < 0.2, -lim, np.where(rng.random(pt.n) < 0.05, lim, pt.req[d]))
    nt.alloc[1] = np.where(rng.random(nt.n) < 0.2, -(1 << 20), nt.alloc[1])
    for shape in ("default", "binpack", "falling", "full"):
        _check_rows(pkg, snap, 16, (1, 0, 1), (1 << 10, SHAPES[shape], [5, 1, 7, 0, 9, 2, 3, 0, 1], 3), seed=991)


def test_zero_weight_is_the_engine_without_it(pkg, oracle):
    snap = random_snapshot(992, P=300, N=800, G=30, L=6, aff=2)
    nz = S.nonzero_requests(snap, 992)
    plain = _rows(pkg, snap, 9, (1, 0, 1), None, nz)
    zero = _rows(pkg, snap, 9, (1, 0, 1), (0, rr.BIN_PACK, [1, 1, 1, 0, 1, 1], 1), nz)
    eng = pkg.Engine(snap.lanes, 0, priority_k=9)
    try:
        eng.upload(snap)
        eng.upload_nonzero(node=nz[0], pods=nz[1])
        eng.set_ratio_priority(4, rr.BIN_PACK, [1, 1, 1, 0, 1, 1], 1)
        eng.evaluate()
        on = eng.priority_rows()
        eng.set_ratio_priority(0, rr.BIN_PACK, [1, 1, 1, 0, 1, 1], 1)
        eng.evaluate()
        off = eng.priority_rows()
    finally:
        eng.close()
    for got in (zero, off):
        np.testing.assert_array_equal(got[0], plain[0])
        np.testing.assert_array_equal(got[1], plain[1])
    assert (on[1] != plain[1]).any()
    want = priority_ref.priority_rows(snap, nz[0], nz[1], 9)
    np.testing.assert_array_equal(plain[0], want[0])


def test_invalid_settings_keep_the_previous_one(pkg, oracle):
    c = pkg.capi
    snap = random_snapshot(993, P=120, N=300, G=10, L=6)
    nz = S.nonzero_requests(snap, 993)
    good = (2, rr.BIN_PACK, [1, 1, 0, 0, 3, 0], 1)
    bad = [dict(shape=((10, 5), (10, 6))), dict(shape=((20, 5), (10, 6))), dict(shape=((0, 5), (101, 6))),
           dict(shape=((0, 101),)), dict(shape=()), dict(shape=tuple((u, 0) for u in range(101)) + ((100, 1),)),
           dict(lw=[1, 1, 0, 1, 0, 0]), dict(lw=[1, 1, 0, 0, 0]), dict(lw=[1, 1, 0, 0, 0, 0, 0]),
           dict(lw=[1 << 23, 1 << 23, 0, 0, 0, 0], absent=1)]
    eng = pkg.Engine(snap.lanes, 0, priority_k=8)
    try:
        eng.upload(snap)
        eng.upload_nonzero(node=nz[0], pods=nz[1])
        eng.set_ratio_priority(*good)
        eng.set_ratio_priority(1, rr.BIN_PACK, [1 << 23, 1 << 23, 0, 0, 0, 0], 0)   # exactly 2^24 is accepted
        eng.set_ratio_priority(*good)
        for b in bad:
            with pytest.raises(c.BsError) as ei:
                eng.set_ratio_priority(5, b.get("shape", rr.DEFAULT_SHAPE), b.get("lw", [1, 0, 0, 0, 0, 0]),
                                       b.get("absent", 0))
            assert ei.value.code == c.BS_E_INVAL, b
        eng.evaluate()
        got = eng.priority_rows()
    finally:
        eng.close()
    want = rr.priority_rows(snap, nz[0], nz[1], 8, good)
    np.testing.assert_array_equal(got[0], want[0])
    np.testing.assert_array_equal(got[1], want[1])


# ---- bs_replay_priority ----
def walk_both(pkg, snap, ratio, weights=(1, 0, 1), queue=None, seed=0, nz=None):
    node_nz, pod_nz = S.nonzero_requests(snap, seed) if nz is None else nz
    eng = pkg.Engine(snap.lanes)
    try:
        eng.upload(snap)
        eng.upload_nonzero(node=node_nz, pods=pod_nz)
        eng.set_score_weights(*weights)
        eng.set_ratio_priority(*ratio)
        got = eng.replay(queue, priority=True)
    finally:
        eng.close()
    pf, node, ready, after, nz_after = rr.replay_ratio(snap, node_nz, pod_nz, ratio, queue, weights)
    np.testing.assert_array_equal(got["prefilter"], pf)
    np.testing.assert_array_equal(got["node"], node)
    np.testing.assert_array_equal(got["ready"], ready)
    nt, gt = after.nodes, after.groups
    want = dict(node_requested=nt.requested, node_pod_count=nt.pod_count, node_req_present=nt.req_present,
                group_matched=gt.matched, group_flags=gt.flags, group_min_res=gt.min_res,
                group_min_res_present=gt.min_res_present, group_rep_sel=gt.rep_sel, group_rep_tol=gt.rep_tol)
    for k in AFTER:
        np.testing.assert_array_equal(got[k], want[k], err_msg=k)
    np.testing.assert_array_equal(got["node_nonzero"], nz_after)
    return got


@pytest.mark.parametrize("seed", range(9))
def test_replay_random(pkg, oracle, seed):
    L = [5, 9, 16][seed % 3]
    snap = random_snapshot(1300 + seed, P=300, N=[70, 1500, 2600][seed // 3], G=40, L=L, case=["mixed", "A", "B"][seed % 3])
    queue = None if seed % 2 == 0 else np.random.default_rng(seed).permutation(snap.pods.n)
    shape = list(SHAPES.values())[seed % len(SHAPES)]
    walk_both(pkg, snap, (1 + seed % 3, shape, _lane_weights(L, seed), seed % 2), WEIGHTS[seed % 3], queue, seed)


def test_replay_negative_values(pkg, oracle):
    snap = random_snapshot(1351, P=300, N=1200, G=20, L=6)
    nt, pt = snap.nodes, snap.pods
    rng = np.random.default_rng(1351)
    nt.alloc[2] = np.where(rng.random(nt.n) < 0.3, -(1 << 40), nt.alloc[2])
    pt.req[2] = np.where(rng.random(pt.n) < 0.3, -(1 << 30), pt.req[2])
    pt.req[4] = np.where(rng.random(pt.n) < 0.2, -(1 << 50), pt.req[4])
    walk_both(pkg, snap, (3, SHAPES["falling"], [1, 1, 2, 0, 5, 1], 1), (1, 0, 1), None, 1351)


def test_replay_first_pass_is_the_round_entry(pkg, oracle):
    snap = random_snapshot(1361, P=300, N=1500, G=30, L=6, case="mixed")
    nz = S.nonzero_requests(snap, 1361)
    ratio = (2, rr.BIN_PACK, [1, 1, 0, 0, 3, 1], 1)
    queue = np.random.default_rng(1361).permutation(snap.pods.n)
    got = walk_both(pkg, snap, ratio, (1, 0, 1), queue, nz=nz)
    first = int(np.flatnonzero(got["prefilter"] == S.PF_PASS)[0])
    nodes, _ = _rows(pkg, snap, 1, (1, 0, 1), ratio, nz)
    assert got["node"][first] == nodes[queue[first], 0]


def test_replay_cfg4_third_scale(pkg, oracle, snapshot_mod):
    snap = snapshot_mod.config(4, scale=0.3)
    eng = pkg.Engine(snap.lanes, fit_bitmap=False, score=False)
    eng.upload(snap)
    order = eng.evaluate().order.copy()
    eng.close()
    lw = [1, 1, 0, 0, 3] + [0] * (snap.lanes - 5)
    got = walk_both(pkg, snap, (1, rr.BIN_PACK, lw, 0), (0, 0, 0), order, seed=4)
    assert got["ready"].sum() > 1000


def test_replay_errors_still_hold(pkg):
    c = pkg.capi
    snap = random_snapshot(1371, P=50, N=80, G=5, L=6)
    node_nz, pod_nz = S.nonzero_requests(snap, 1371)
    eng = pkg.Engine(snap.lanes)
    try:
        eng.upload(snap)
        eng.set_ratio_priority(1, rr.BIN_PACK, [1, 1, 1, 0, 1, 1], 0)
        with pytest.raises(c.BsError) as ei:
            eng.replay(priority=True)
        assert ei.value.code == c.BS_E_STATE
        big = np.full((2, snap.pods.n), c.NONZERO_MAX, np.int64)
        eng.upload_nonzero(node=np.full((2, snap.nodes.n), c.NONZERO_MAX, np.int64), pods=big)
        eng.replay(np.arange(63, dtype=np.uint32) % snap.pods.n, priority=True)
        with pytest.raises(c.BsError) as ei:
            eng.replay(np.arange(64, dtype=np.uint32) % snap.pods.n, priority=True)
        assert ei.value.code == c.BS_E_RANGE
    finally:
        eng.close()


def test_plugin_ratio_priority(pkg, tmp_path):
    """BatchSchedulingPlugin::SetRatioPriority through tests/cpp/plugin_ratio_priority_test.cpp: the lane mapping over
    two rounds whose scalar lanes come in different orders, pods and unknown names in absent_weight, the x10 scaling,
    and PriorityNodes / ReplayQueue(kPriority) equal to the engine called directly."""
    pkg.capi.load()
    src = os.path.join(ROOT, "tests", "cpp", "plugin_ratio_priority_test.cpp")
    libdir = os.path.join(ROOT, "batch-scheduler_b200")
    binary = str(tmp_path / "plugin_ratio_priority_test")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-o", binary, src, "-L" + libdir, "-lbsched",
                           "-Wl,-rpath," + libdir, "-L/usr/local/cuda/lib64", "-Wl,-rpath,/usr/local/cuda/lib64"])
    o = json.loads(subprocess.check_output([binary], text=True))
    for r in o["rounds"]:
        assert r["plugin_nodes"] == r["engine_nodes"] and r["plugin_scores"] == r["engine_scores"], r
        assert r["plugin_replay"] == r["engine_replay"], r
    # round 1: gpu is lane 5 (foo came first); round 2: gpu is lane 4
    assert o["rounds"][0]["gpu_lane"] == 5 and o["rounds"][1]["gpu_lane"] == 4
    # bin-pack by GPU: the pod goes to the busier GPU node (node-1), in both rounds
    assert [r["plugin_nodes"][0] for r in o["rounds"]] == ["node-1", "node-1"]
    assert o["invalid_shape_fails"] == 1
