"""GPU: the ImageLocality and NodePreferAvoidPods priorities (bs_set_locality_weights) in the round's priority lists and
in bs_replay_priority, bit-exact against the CPU restatement tests/locality_priority_ref.c: every lane build, list
lengths, unaligned sizes, four weight pairs with the ratio term and the node priorities on and off; the walk and its
after-state; weights (0, 0) are the engine without them; the other outputs do not move; the node side follows
bs_update_nodes; every error code; sampled pods at cfg4 size; and the C++ plugin's SetLocalityWeights over objects."""
import numpy as np
import pytest

import locality_priority_ref as lr
import node_priority_ref as npr
import ratio_priority_ref as rr
from randsnap import S, random_snapshot

pytestmark = pytest.mark.gpu

LW = [(1, 0), (0, 10000), (1, 10000), (3, 7)]
PW = (1, 1)


def _ratio(L, on):
    return (2, rr.BIN_PACK, [1, 1, 0, 0] + [1] * (L - 4), 1) if on else npr.NO_RATIO


def _engine(pkg, snap, K, nz, loc, lw, ratio=None, prefs=None, weights=(1, 0, 1), **kw):
    eng = pkg.Engine(snap.lanes, 0, priority_k=K, **kw)
    eng.upload(snap)
    eng.upload_nonzero(node=nz[0], pods=nz[1])
    eng.set_score_weights(*weights)
    if ratio is not None and ratio[0]:
        eng.set_ratio_priority(*ratio)
    if prefs is not None:
        eng.upload_preferences(node=(prefs[0], prefs[1]), pods=(prefs[2], prefs[3]))
        eng.set_node_priority_weights(*PW)
    if loc is not None:
        eng.upload_locality(node=loc[0], pods=loc[1])
    eng.set_locality_weights(*lw)
    return eng


def _check(pkg, snap, K, lw, ratio_on, pref_on, seed, weights=(1, 0, 1), loc=None):
    nz = S.nonzero_requests(snap, seed)
    loc = S.node_locality(snap, seed) if loc is None else loc
    prefs = S.node_preferences(snap, seed) if pref_on else None
    ratio = _ratio(snap.lanes, ratio_on)
    eng = _engine(pkg, snap, K, nz, loc, lw, ratio, prefs, weights)
    try:
        eng.evaluate()
        nodes, scores = eng.priority_rows()
    finally:
        eng.close()
    want_n, want_s = lr.priority_rows(snap, nz[0], nz[1], K, loc, lw, ratio, weights, prefs, PW)
    np.testing.assert_array_equal(nodes, want_n)
    np.testing.assert_array_equal(scores, want_s)
    return nodes, scores


@pytest.mark.parametrize("L", [5, 9, 16])
@pytest.mark.parametrize("lw", LW)
@pytest.mark.parametrize("ratio_on", [False, True])
@pytest.mark.parametrize("pref_on", [False, True])
def test_lane_builds(pkg, oracle, L, lw, ratio_on, pref_on):
    snap = random_snapshot(1400 + L, P=200, N=500, G=30, L=L, case="mixed")
    K = {5: 1, 9: 7, 16: 32}[L]
    _check(pkg, snap, K, lw, ratio_on, pref_on, seed=L)


@pytest.mark.parametrize("K", [1, 7, 32])
@pytest.mark.parametrize("lw", LW)
def test_lengths_and_weights(pkg, oracle, K, lw):
    snap = random_snapshot(1450 + K, P=300, N=900, G=30, L=6, aff=3)
    _check(pkg, snap, K, lw, K == 7, K == 32, seed=K, weights=(2, 1, 3))


@pytest.mark.parametrize("P,N", [(1, 1), (37, 31), (70, 33), (131, 511), (95, 1025)])
def test_unaligned_sizes(pkg, oracle, P, N):
    snap = random_snapshot(P * 5 + N, P=P, N=N, G=9, L=6)
    _check(pkg, snap, 7, (1, 10000), N % 2 == 1, False, seed=N)


def test_hand_thresholds_on_device(pkg, oracle):
    """Sums on both thresholds and the binary64 case of the scaling, through the device pre-pass."""
    MIB = 1 << 20
    snap = random_snapshot(1460, P=40, N=100, G=5, L=5)
    N = snap.nodes.n
    rows = np.zeros((5, N), bool)
    rows[0] = True                    # 23 MiB everywhere
    rows[1] = True                    # 1000 MiB everywhere
    rows[2, :29] = True               # 100 MiB on 29 of 100 nodes: scaled 30408703
    rows[3, :50] = True               # 2000 MiB on half the nodes: scaled 1000 MiB
    rows[4, ::3] = True
    sizes = [23 * MIB, 1000 * MIB, 100 * MIB, 2000 * MIB, 400 * MIB]
    W = (N + 31) // 32
    pad = np.zeros((5, W * 32), bool)
    pad[:, :N] = rows
    bits = (pad.reshape(5, W, 32).astype(np.uint64) << np.arange(32, dtype=np.uint64)).sum(
        axis=2, dtype=np.uint64).astype(np.uint32)
    classes = [[0], [1], [2, 2, 2], [3], [4, 4], [0, 2]]
    off = np.concatenate([[0], np.cumsum([len(c) for c in classes])]).astype(np.uint32)
    ids = np.array([i for c in classes for i in c], np.uint32)
    cls = (np.arange(snap.pods.n) % 7).astype(np.uint32)
    cls[cls == 6] = S.IMAGE_NONE
    loc = ((np.array(sizes, np.int64), bits, np.zeros(N, np.uint64)),
           (cls, off, ids, np.full(snap.pods.n, S.AVOID_NONE, np.uint8)))
    assert lr.scaled(loc, N).tolist()[2:4] == [30408703, 1000 * MIB]
    _check(pkg, snap, 32, (1, 0), False, False, seed=3, loc=loc)


def test_zero_weights_are_the_engine_without_them(pkg, oracle):
    snap = random_snapshot(1461, P=300, N=800, G=30, L=6, aff=2)
    nz = S.nonzero_requests(snap, 1461)
    loc = S.node_locality(snap, 1461)
    out, walks = [], []
    for with_cols in (False, True):
        eng = _engine(pkg, snap, 9, nz, loc if with_cols else None, (0, 0))
        try:
            eng.evaluate()
            out.append(eng.priority_rows())
            walks.append(eng.replay(priority=True))
            if with_cols:   # on, then off again on the same engine
                eng.set_locality_weights(1, 10000)
                eng.evaluate()
                on = eng.priority_rows()
                eng.set_locality_weights(0, 0)
                eng.evaluate()
                out.append(eng.priority_rows())
                walks.append(eng.replay(priority=True))
        finally:
            eng.close()
    for nodes, scores in out[1:]:
        np.testing.assert_array_equal(nodes, out[0][0])
        np.testing.assert_array_equal(scores, out[0][1])
    for w in walks[1:]:
        for k, v in walks[0].items():
            np.testing.assert_array_equal(w[k], v, err_msg=k)
    assert not np.array_equal(on[1], out[0][1])


def test_other_outputs_do_not_move(pkg, oracle):
    snap = random_snapshot(1462, P=300, N=800, G=30, L=6)
    nz = S.nonzero_requests(snap, 1462)
    loc = S.node_locality(snap, 1462)
    got = []
    for lw in ((0, 0), (3, 7)):
        eng = _engine(pkg, snap, 8, nz, loc, lw, fit_bitmap=True, topk=8, reasons=True)
        try:
            res = eng.evaluate()
            got.append((res, eng.fit_rows(), eng.topk_rows(), eng.reason_rows()))
        finally:
            eng.close()
    (r0, f0, t0, q0), (r1, f1, t1, q1) = got
    for f in ("prefilter", "feasible_count", "best_node", "best_score", "admit", "order", "rank"):
        np.testing.assert_array_equal(getattr(r0, f), getattr(r1, f), err_msg=f)
    np.testing.assert_array_equal(f0, f1)
    np.testing.assert_array_equal(t0[0], t1[0])
    np.testing.assert_array_equal(t0[1], t1[1])
    np.testing.assert_array_equal(q0, q1)


@pytest.mark.parametrize("seed", range(4))
def test_replay_priority(pkg, oracle, seed):
    """bs_replay_priority with the terms: placements, readiness and the after-state equal the hooked CPU walk."""
    snap = random_snapshot(1470 + seed, P=120, N=[60, 300][seed % 2], G=20, L=[5, 6, 9, 16][seed], case="mixed")
    nz = S.nonzero_requests(snap, seed)
    loc = S.node_locality(snap, seed, avoided=0.4)
    lw = LW[seed]
    ratio = _ratio(snap.lanes, seed % 2 == 1)
    queue = None if seed % 2 == 0 else np.random.default_rng(seed).permutation(snap.pods.n).astype(np.uint32)
    eng = _engine(pkg, snap, 4, nz, loc, lw, ratio)
    try:
        res = eng.replay(queue, priority=True)
    finally:
        eng.close()
    pf, node, ready, after, live = lr.replay_locality(snap, nz[0], nz[1], loc, lw, ratio, queue)
    np.testing.assert_array_equal(res["prefilter"], pf)
    np.testing.assert_array_equal(res["node"], node)
    np.testing.assert_array_equal(res["ready"], ready)
    nt, gt = after.nodes, after.groups
    want = dict(node_requested=nt.requested, node_pod_count=nt.pod_count, node_req_present=nt.req_present,
                group_matched=gt.matched, group_flags=gt.flags, group_min_res=gt.min_res,
                group_min_res_present=gt.min_res_present, group_rep_sel=gt.rep_sel, group_rep_tol=gt.rep_tol)
    for k, v in want.items():
        np.testing.assert_array_equal(res[k], v, err_msg=k)
    np.testing.assert_array_equal(res["node_nonzero"], live)
    assert (node >= 0).any()


def test_node_side_follows_row_updates(pkg, oracle):
    c = pkg.capi
    snap = random_snapshot(1480, P=200, N=500, G=20, L=6)
    nz = S.nonzero_requests(snap, 1480)
    loc = S.node_locality(snap, 1480)
    eng = _engine(pkg, snap, 16, nz, loc, (1, 10000))
    try:
        eng.evaluate()
        idx = np.arange(0, snap.nodes.n, 7)
        eng.update_nodes(idx, snap.nodes.take(idx))
        eng.upload_nonzero(node=nz[0])
        with pytest.raises(c.BsError) as ei:
            eng.evaluate()
        assert ei.value.code == c.BS_E_STATE
        with pytest.raises(c.BsError) as ei:
            eng.replay(priority=True)
        assert ei.value.code == c.BS_E_STATE
        (size, bits, avoid), pods = loc
        bits2, avoid2 = bits.copy(), avoid.copy()
        bits2[:, 0] ^= np.uint32(0xFFFF)     # nodes 0-15 report the other names now
        avoid2[idx] = np.uint64(0xFF)
        loc2 = ((size, bits2, avoid2), pods)
        eng.upload_locality(node=loc2[0])
        eng.evaluate()
        nodes, scores = eng.priority_rows()
    finally:
        eng.close()
    want_n, want_s = lr.priority_rows(snap, nz[0], nz[1], 16, loc2, (1, 10000))
    np.testing.assert_array_equal(nodes, want_n)
    np.testing.assert_array_equal(scores, want_s)


def test_errors(pkg):
    c = pkg.capi
    snap = random_snapshot(1490, P=50, N=80, G=5, L=6)
    nz = S.nonzero_requests(snap, 1490)
    (size, bits, avoid), (cls, off, ids, abit) = S.node_locality(snap, 1490)
    lib = c.load()

    def code(f, *a):
        with pytest.raises(c.BsError) as ei:
            f(*a)
        return ei.value.code

    eng = _engine(pkg, snap, 4, nz, None, (0, 0))
    h = eng.h
    try:
        # wrong sizes, a size outside [0, 2^48], an avoid bit outside 0..63, a class over 64 ids, tables over the cap
        assert code(eng.upload_locality, (size, bits, avoid[:-1]), None) == c.BS_E_INVAL
        assert code(eng.upload_locality, None, (cls[:-1], off, ids, abit[:-1])) == c.BS_E_INVAL
        big = size.copy()
        big[2] = c.IMAGE_SIZE_MAX + 1
        assert code(eng.upload_locality, (big, bits, avoid), None) == c.BS_E_RANGE
        big[2] = -1
        assert code(eng.upload_locality, (big, bits, avoid), None) == c.BS_E_RANGE
        bad_bit = abit.copy()
        bad_bit[3] = 64
        assert code(eng.upload_locality, None, (cls, off, ids, bad_bit)) == c.BS_E_RANGE
        long_off = np.array([0, 65], np.uint32)
        assert code(eng.upload_locality, None, (np.zeros(snap.pods.n, np.uint32), long_off,
                                                np.zeros(65, np.uint32), abit)) == c.BS_E_INVAL
        words = (snap.nodes.n + 31) // 32
        n_img = c.LOC_TABLE_MAX_BYTES // (words * 4) + 1
        assert lib.bs_upload_node_locality(h, snap.nodes.n, n_img, c.ptr(size), c.ptr(bits), None) == c.BS_E_INVAL
        n_cls = c.LOC_TABLE_MAX_BYTES // (((snap.nodes.n + 31) // 32) * 32) + 1
        assert lib.bs_upload_pod_locality(h, snap.pods.n, c.ptr(cls), n_cls, c.ptr(off), c.ptr(ids), None) == c.BS_E_INVAL
        # missing columns: BS_E_STATE before anything launches, per weight, in the round and in the walk
        eng.set_locality_weights(1, 0)
        assert code(eng.evaluate) == c.BS_E_STATE
        assert code(lambda: eng.replay(priority=True)) == c.BS_E_STATE
        eng.upload_locality(pods=(cls, off, ids, abit))
        assert code(eng.evaluate) == c.BS_E_STATE    # the node side failed above: still missing
        eng.upload_locality(node=(None, None, avoid))
        assert code(eng.evaluate) == c.BS_E_STATE    # the image part of the node side is missing
        eng.upload_locality(node=(size, bits, None))
        eng.evaluate()
        eng.replay(priority=True)
        eng.set_locality_weights(1, 1)
        assert code(eng.evaluate) == c.BS_E_STATE    # now the avoid part is missing
        eng.upload_locality(node=(size, bits, avoid))
        eng.evaluate()
        eng.upload(snap)                             # new pods and nodes drop both sides
        eng.upload_nonzero(node=nz[0], pods=nz[1])
        assert code(eng.evaluate) == c.BS_E_STATE
        eng.set_locality_weights(0, 1)
        eng.upload_locality(node=(None, None, avoid), pods=(None, None, None, abit))
        eng.evaluate()
        eng.replay(priority=True)
        # ids outside the tables: BS_E_INDEX at evaluation (only where the ImageLocality weight reads them)
        eng.set_locality_weights(1, 1)
        eng.upload_locality(node=(size, bits, avoid))
        bad = cls.copy()
        bad[5] = len(off) - 1
        eng.upload_locality(pods=(bad, off, ids, abit))
        assert code(eng.evaluate) == c.BS_E_INDEX
        assert code(lambda: eng.replay(priority=True)) == c.BS_E_INDEX
        bad_ids = ids.copy()
        bad_ids[0] = len(size)
        eng.upload_locality(pods=(cls, off, bad_ids, abit))
        assert code(eng.evaluate) == c.BS_E_INDEX
        eng.set_locality_weights(0, 1)
        eng.evaluate()
        eng.set_locality_weights(1, 1)
        eng.upload_locality(pods=(cls, off, ids, abit))
        eng.evaluate()
        # TaintToleration / NodeAffinity still refuse the walk
        eng.set_node_priority_weights(1, 0)
        assert code(lambda: eng.replay(priority=True)) == c.BS_E_INVAL
    finally:
        eng.close()


def test_full_size_cfg4(pkg, oracle, snapshot_mod):
    snap = snapshot_mod.config(4)
    nz = snapshot_mod.nonzero_requests(snap, 4)
    loc = snapshot_mod.node_locality(snap, 4)
    eng = _engine(pkg, snap, 16, nz, loc, (1, 10000), fit_bitmap=False)
    try:
        res = eng.evaluate()
        nodes, scores = eng.priority_rows()
    finally:
        eng.close()
    idx = np.sort(np.random.default_rng(4).choice(snap.pods.n, 200, replace=False))
    want_n, want_s = lr.priority_rows(snap, nz[0], nz[1], 16, loc, (1, 10000), pods=idx)
    np.testing.assert_array_equal(nodes[idx], want_n)
    np.testing.assert_array_equal(scores[idx], want_s)
    np.testing.assert_array_equal((nodes >= 0).sum(axis=1), np.minimum(16, res.feasible_count))


def test_plugin_locality_weights():
    """The C++ plugin's SetLocalityWeights(1, 10000) over objects: PriorityNodes and ReplayQueue(kPriority) equal an
    engine called directly with PackLocality's columns, and the avoided nodes rank last for the controlled pods."""
    import json
    import subprocess

    import native
    o = json.loads(subprocess.check_output([native.cpp_program("plugin_locality_priority_test"), "gpu"], text=True))
    assert o["plugin"] == o["engine"]
    assert o["plugin_replay"] == o["engine_replay"]
    last = {p: [n for n, _ in o["plugin"][p]] for p in range(len(o["pods"]))}
    assert set(last[0][-2:]) == {"node-0", "node-4"}   # ReplicaSet rs-1 is avoided there
    assert set(last[5][-2:]) == {"node-0", "node-4"}
    assert last[1][-1] == "node-1"                      # ReplicationController rc-1
    assert last[3][-1] == "node-2"                      # ReplicaSet rs-2
    assert len(last[2]) == len(o["nodes"])              # a StatefulSet counts as no controller: nothing is avoided
    scores2 = [s for _, s in o["plugin"][2]]
    assert max(scores2) - min(scores2) < 10000 * 100
