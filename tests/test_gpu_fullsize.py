"""GPU, BASELINE.json's full sizes: bit-exact decisions against the (multi-threaded) oracle where the
oracle finishes in seconds, and size-independent properties of the materialised matrices elsewhere."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _popcount_rows(words):
    return np.unpackbits(words.view(np.uint8), axis=1).sum(axis=1).astype(np.uint32)


def _properties(snap, res, eng, S, sample_rows=64):
    P, N, G = snap.pods.n, snap.nodes.n, snap.groups.n
    # order is a permutation, rank is monotone along it and dense
    assert np.array_equal(np.sort(res.order), np.arange(P, dtype=np.uint32))
    r_along = res.rank[res.order]
    assert (np.diff(r_along.astype(np.int64)) >= 0).all() and (np.diff(r_along.astype(np.int64)) <= 1).all()
    assert r_along[0] == 0
    # Compare's leading key: priority never increases along the order
    assert (np.diff(snap.pods.priority[res.order].astype(np.int64)) <= 0).all()
    # admit bitmap <-> admit codes
    bits = np.unpackbits(res.admit_bitmap.view(np.uint8), bitorder="little")[:G]
    assert np.array_equal(bits.astype(bool), res.admit == S.ADMIT)
    # new_denied only for groups with a NOT_ENOUGH pod, and every such group is flagged
    ne = res.prefilter == S.PF_NOT_ENOUGH
    flagged = np.zeros(G, bool)
    flagged[snap.pods.gid[ne]] = True
    assert np.array_equal(flagged, res.new_denied.astype(bool))
    # Permit readiness recomputed from the per-pod outputs (core.go:303, uint32)
    ok = (res.prefilter == S.PF_PASS) & (res.feasible_count > 0) & (snap.pods.gid >= 0)
    contrib = np.bincount(snap.pods.gid[ok], minlength=G).astype(np.uint32)
    in_round = np.bincount(snap.pods.gid[snap.pods.gid >= 0], minlength=G)
    need = (snap.groups.min_member - snap.groups.scheduled).astype(np.uint32)
    ready = (snap.groups.matched + contrib).astype(np.uint32) >= need
    exp = np.where((in_round > 0) & (contrib == 0), S.UNSCHEDULABLE, np.where(ready, S.ADMIT, S.WAIT))
    assert np.array_equal(exp.astype(np.uint8), res.admit)
    # sampled rows of the matrices: bitmap popcount, score sign, best node
    rows = np.linspace(0, P - 1, sample_rows).astype(int)
    for p in rows:
        w = eng.fit_rows(int(p), 1)
        sc = eng.score_rows(int(p), 1)[0]
        fit = np.unpackbits(w.view(np.uint8), bitorder="little")[:N].astype(bool)
        assert fit.sum() == res.feasible_count[p]
        assert ((sc >= 0) == fit).all() and (sc[~fit] == np.iinfo(np.int64).min).all()
        if fit.any():
            assert res.best_score[p] == sc.max() and res.best_node[p] == int(np.argmax(sc))
        else:
            assert res.best_node[p] == -1


@pytest.mark.parametrize("cfg", [3, 4])
def test_full_size_decisions_and_properties(pkg, oracle, snapshot_mod, cfg):
    S = snapshot_mod
    snap = S.config(cfg)
    eng = pkg.Engine(snap.lanes, 0, fit_bitmap=True, score=True)
    eng.upload(snap)
    res = eng.evaluate()
    _properties(snap, res, eng, S)
    orc = oracle.round(snap, want_bitmap=False, want_score=False, threads=0)
    for f in ("prefilter", "feasible_count", "best_node", "best_score", "admit", "admit_bitmap", "new_denied",
              "order", "rank"):
        np.testing.assert_array_equal(getattr(res, f), getattr(orc, f), err_msg=f)
    assert res.max_group == orc.max_group
    # a slice of the matrices against the oracle
    sub = S.Snapshot(snap.nodes, snap.pods.take(np.arange(2000, 2300)), snap.groups)
    o2 = oracle.round(sub, want_bitmap=True, want_score=True, want_sort=False)
    np.testing.assert_array_equal(eng.fit_rows(2000, 300), o2.fit_bitmap)
    np.testing.assert_array_equal(eng.score_rows(2000, 300), o2.score)
    eng.close()


def test_cfg5_one_rank_shard_full_size(pkg, oracle, snapshot_mod):
    """BASELINE configs[4] (1M pods / 50k nodes / 62.5k groups / 9 lanes) as rank 0 of the 8-way group sharding sees
    it: 125k pods x ALL 50k nodes, a 50 GB int64 score shard + fit bitmap on one GPU.  Every decision vector against
    the multi-threaded oracle round on the same shard, 300 rows of both matrices, and the size-independent properties."""
    import torch
    if torch.cuda.mem_get_info()[0] < 60e9:
        pytest.skip("needs ~55 GB of free HBM")
    S = snapshot_mod
    full = S.config(5).resolve_groups()
    snap = full.shard_groups(0, 8)
    assert 124900 <= snap.pods.n <= 125100 and snap.nodes.n == 50000 and snap.lanes == 9   # ranges follow group borders
    eng = pkg.Engine(snap.lanes, 0, fit_bitmap=True, score=True)
    eng.upload(snap)
    res = eng.evaluate()
    assert eng.fit_shape()["LW"] + eng.fit_shape()["LN"] + eng.fit_shape()["LS"] == 9
    _properties(snap, res, eng, S, sample_rows=16)
    orc = oracle.round(snap, want_bitmap=False, want_score=False, threads=0)
    for f in ("prefilter", "feasible_count", "best_node", "best_score", "admit", "admit_bitmap", "new_denied",
              "order", "rank"):
        np.testing.assert_array_equal(getattr(res, f), getattr(orc, f), err_msg=f)
    assert res.max_group == orc.max_group and res.max_finished == orc.max_finished
    for p0 in (0, 62000, 124900):
        sub = S.Snapshot(snap.nodes, snap.pods.take(np.arange(p0, p0 + 100)), snap.groups)
        o2 = oracle.round(sub, want_bitmap=True, want_score=True, want_sort=False)
        np.testing.assert_array_equal(eng.fit_rows(p0, 100), o2.fit_bitmap)
        np.testing.assert_array_equal(eng.score_rows(p0, 100), o2.score)
    eng.close()


def test_replay_full_size_conservation(pkg, snapshot_mod):
    """bs_replay on BASELINE configs[3] at full size (100k pods in device-sort order): properties that
    hold for any correct walk — every debit is accounted for, a pod is only assumed after passing
    PreFilter, gangs are flagged exactly when Permit's uint32 compare says so, refused groups freeze."""
    S = snapshot_mod
    snap = S.config(4)
    P, N, G, L = snap.pods.n, snap.nodes.n, snap.groups.n, snap.lanes
    eng = pkg.Engine(L, 0, fit_bitmap=False, score=False)
    eng.upload(snap)
    order = eng.evaluate().order.copy()
    out = eng.replay(order)
    eng.close()
    pf, node, ready = out["prefilter"], out["node"], out["ready"]
    pods = order
    placed = node >= 0
    assert (pf[placed] == S.PF_PASS).all() and placed.sum() > 10000
    # requested grew by exactly the requests of the pods assumed onto each node (pods lane: pod list)
    for d in range(L):
        if d == 3:
            continue
        add = np.zeros(N, np.int64)
        use = placed & ((d < 4) | (((snap.pods.req_present[pods] >> np.uint32(d)) & 1) == 1))
        np.add.at(add, node[use], snap.pods.req[d, pods[use]])
        np.testing.assert_array_equal(out["node_requested"][d], snap.nodes.requested[d] + add)
    np.testing.assert_array_equal(out["node_requested"][3], snap.nodes.requested[3])
    np.testing.assert_array_equal(out["node_pod_count"], snap.nodes.pod_count + np.bincount(node[placed], minlength=N))
    # matched grew by the pods assumed per group; Scheduled <=> the gang completed during the walk
    gid = snap.pods.gid[pods]
    grouped = placed & (gid >= 0)
    np.testing.assert_array_equal(out["group_matched"], snap.groups.matched + np.bincount(gid[grouped], minlength=G).astype(np.uint32))
    newly = (out["group_flags"] & S.GROUP_SCHEDULED) & ~(snap.groups.flags & S.GROUP_SCHEDULED)
    completed = np.zeros(G, bool)
    completed[gid[(ready == 1) & (gid >= 0)]] = True
    assert np.array_equal(newly.astype(bool), completed & ~(snap.groups.flags & S.GROUP_SCHEDULED).astype(bool))
    # a refused group is frozen: after its NOT_ENOUGH pod every later pod of the group is DENIED
    ne_first = {}
    for qi in np.flatnonzero(pf == S.PF_NOT_ENOUGH):
        ne_first.setdefault(int(gid[qi]), int(qi))
    later = np.array([qi > ne_first.get(int(g), P) for qi, g in enumerate(gid)])
    assert (pf[later] == S.PF_DENIED).all() and later.sum() > 1000
    # no node is left over-committed on a lane the walk debited (it only assumes where the pod fits)
    left_cpu = snap.nodes.alloc[0] - out["node_requested"][0]
    touched = np.bincount(node[placed], minlength=N) > 0
    assert (left_cpu[touched] >= 0).all()
