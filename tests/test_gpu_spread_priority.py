"""GPU: the SelectorSpread priority (bs_set_spread_weight) in the round's priority lists, bit-exact against the CPU
restatement tests/spread_priority_ref.c: every lane build, list lengths, unaligned sizes, every combination of the
ratio term, the node priorities and the locality priorities with SPREAD on (the shared first sweep); 0, 1 and 64
zones with zoned and unzoned nodes; counts at BS_SPREAD_COUNT_MAX and the binary64 pins; weight 0 is the engine
without the columns; the other outputs do not move; the drop rules; every error code; the walk's refusal; sampled pods
at cfg4 size."""
import numpy as np
import pytest

import node_priority_ref as npr
import ratio_priority_ref as rr
import spread_priority_ref as sr
from randsnap import S, random_snapshot

pytestmark = pytest.mark.gpu

PW = (1, 1)
LW = (1, 10000)


def _ratio(L, on):
    return (2, rr.BIN_PACK, [1, 1, 0, 0] + [1] * (L - 4), 1) if on else npr.NO_RATIO


def _engine(pkg, snap, K, nz, spread, w, ratio=None, prefs=None, loc=None, weights=(1, 0, 1), **kw):
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
        eng.set_locality_weights(*LW)
    if spread is not None:
        eng.upload_spread(node=spread[0], pods=spread[1])
    eng.set_spread_weight(w)
    return eng


def _check(pkg, snap, K, w, seed, ratio_on=False, pref_on=False, loc_on=False, weights=(1, 0, 1), spread=None,
           n_zones=4):
    nz = S.nonzero_requests(snap, seed)
    spread = S.node_spread(snap, seed, n_zones=n_zones) if spread is None else spread
    prefs = S.node_preferences(snap, seed) if pref_on else None
    loc = S.node_locality(snap, seed) if loc_on else None
    ratio = _ratio(snap.lanes, ratio_on)
    eng = _engine(pkg, snap, K, nz, spread, w, ratio, prefs, loc, weights)
    try:
        eng.evaluate()
        nodes, scores = eng.priority_rows()
    finally:
        eng.close()
    want_n, want_s = sr.priority_rows(snap, nz[0], nz[1], K, spread, w, ratio, weights, prefs,
                                      PW if pref_on else (0, 0), loc, LW if loc_on else (0, 0))
    np.testing.assert_array_equal(nodes, want_n)
    np.testing.assert_array_equal(scores, want_s)
    return nodes, scores


@pytest.mark.parametrize("L", [5, 9, 16])
@pytest.mark.parametrize("ratio_on", [False, True])
@pytest.mark.parametrize("pref_on", [False, True])
@pytest.mark.parametrize("loc_on", [False, True])
def test_flag_combinations(pkg, oracle, L, ratio_on, pref_on, loc_on):
    snap = random_snapshot(2100 + L, P=200, N=500, G=30, L=L, case="mixed")
    K = {5: 1, 9: 7, 16: 32}[L]
    _check(pkg, snap, K, 1, L, ratio_on, pref_on, loc_on)


@pytest.mark.parametrize("K", [1, 7, 32])
@pytest.mark.parametrize("w", [1, 7])
def test_lengths_and_weights(pkg, oracle, K, w):
    snap = random_snapshot(2150 + K, P=300, N=900, G=30, L=6, aff=3)
    _check(pkg, snap, K, w, K, K == 7, K == 32, weights=(2, 1, 3))


@pytest.mark.parametrize("P,N", [(1, 1), (37, 31), (70, 33), (131, 511), (95, 1025)])
def test_unaligned_sizes(pkg, oracle, P, N):
    snap = random_snapshot(P * 5 + N + 2100, P=P, N=N, G=9, L=6)
    _check(pkg, snap, 7, 1, N, N % 2 == 1)


@pytest.mark.parametrize("n_zones", [0, 1, 64])
@pytest.mark.parametrize("unzoned", [0.0, 0.3])
def test_zones(pkg, oracle, n_zones, unzoned):
    snap = random_snapshot(2160 + n_zones, P=200, N=700, G=20, L=5)
    spread = S.node_spread(snap, n_zones, n_zones=n_zones, unzoned=unzoned, occupied=0.5)
    _check(pkg, snap, 16, 1, 3, spread=spread)


def test_counts_at_the_cap_and_the_pins(pkg, oracle):
    """Counts of 2^24 on many nodes of one zone (zone sums far above 2^32), and the two binary64 pins: Mn = 50 with
    count 21 and no zones (57, not 58), and a pod of fit-set-wide selectors."""
    snap = random_snapshot(2170, P=120, N=600, G=20, L=5)
    N = snap.nodes.n
    (zone, counts), cls = S.node_spread(snap, 2170, n_zones=2, unzoned=0.1)
    counts[0] = np.where(np.arange(N) % 3 == 0, 1 << 24, (1 << 24) - 1)
    counts[1] = 0
    counts[1, :N // 2] = 21
    counts[1, N // 2:] = 50   # every pod of class 1 that fits both halves: Mn = 50, count 21
    z1 = np.where(counts[1] > 0, S.ZONE_NONE, 0).astype(np.uint8)
    cls[:40] = 0
    cls[40:80] = 1
    _check(pkg, snap, 32, 1, 1, spread=((zone, counts), cls))
    _check(pkg, snap, 32, 1, 1, spread=((z1, counts), cls))
    ss = sr.ss_matrix(snap, ((np.full(N, S.ZONE_NONE, np.uint8), counts), cls), range(40, 80))
    full = ss[(ss[:, :N // 2] >= 0).any(axis=1) & (ss[:, N // 2:] >= 0).any(axis=1)]
    if len(full):
        assert 57 in full[:, :N // 2]


def test_zero_weight_is_the_engine_without_columns(pkg, oracle):
    snap = random_snapshot(2180, P=300, N=800, G=30, L=6, aff=2)
    nz = S.nonzero_requests(snap, 2180)
    spread = S.node_spread(snap, 2180)
    out = []
    for with_cols in (False, True):
        eng = _engine(pkg, snap, 9, nz, spread if with_cols else None, 0)
        try:
            eng.evaluate()
            out.append(eng.priority_rows())
            if with_cols:   # on, then off again on the same engine
                eng.set_spread_weight(1)
                eng.evaluate()
                on = eng.priority_rows()
                eng.set_spread_weight(0)
                eng.evaluate()
                out.append(eng.priority_rows())
        finally:
            eng.close()
    for nodes, scores in out[1:]:
        np.testing.assert_array_equal(nodes, out[0][0])
        np.testing.assert_array_equal(scores, out[0][1])
    assert not np.array_equal(on[1], out[0][1])


def test_other_outputs_do_not_move(pkg, oracle):
    snap = random_snapshot(2181, P=300, N=800, G=30, L=6)
    nz = S.nonzero_requests(snap, 2181)
    spread = S.node_spread(snap, 2181)
    got = []
    for w in (0, 3):
        eng = _engine(pkg, snap, 8, nz, spread, w, fit_bitmap=True, topk=8, reasons=True)
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


def test_drop_rules(pkg, oracle):
    """bs_update_nodes drops the node side, bs_upload_pods the pod side; uploading them again restores the lists."""
    c = pkg.capi
    snap = random_snapshot(2182, P=200, N=500, G=20, L=6)
    nz = S.nonzero_requests(snap, 2182)
    (zone, counts), cls = S.node_spread(snap, 2182)
    eng = _engine(pkg, snap, 16, nz, ((zone, counts), cls), 1)
    try:
        eng.evaluate()
        idx = np.arange(0, snap.nodes.n, 7)
        eng.update_nodes(idx, snap.nodes.take(idx))
        eng.upload_nonzero(node=nz[0])
        with pytest.raises(c.BsError) as ei:
            eng.evaluate()
        assert ei.value.code == c.BS_E_STATE
        counts2 = counts.copy()
        counts2[:, idx] += 3   # pods bound on the changed nodes
        eng.upload_spread(node=(zone, counts2))
        eng.evaluate()
        nodes, scores = eng.priority_rows()
        eng.upload(snap)   # the pod table again: both sides go
        eng.upload_nonzero(node=nz[0], pods=nz[1])
        eng.upload_spread(node=(zone, counts2))
        with pytest.raises(c.BsError) as ei:
            eng.evaluate()
        assert ei.value.code == c.BS_E_STATE
        eng.upload_spread(pods=cls)
        eng.evaluate()
        nodes2, scores2 = eng.priority_rows()
    finally:
        eng.close()
    want_n, want_s = sr.priority_rows(snap, nz[0], nz[1], 16, ((zone, counts2), cls), 1)
    for n, s in ((nodes, scores), (nodes2, scores2)):
        np.testing.assert_array_equal(n, want_n)
        np.testing.assert_array_equal(s, want_s)


def test_errors_and_the_walk(pkg):
    c = pkg.capi
    snap = random_snapshot(2190, P=50, N=80, G=5, L=6)
    nz = S.nonzero_requests(snap, 2190)
    (zone, counts), cls = S.node_spread(snap, 2190, n_zones=3)
    lib = c.load()
    N = snap.nodes.n

    def code(f, *a, **kw):
        with pytest.raises(c.BsError) as ei:
            f(*a, **kw)
        return ei.value.code

    eng = _engine(pkg, snap, 4, nz, None, 0)
    h = eng.h
    try:
        eng.evaluate()
        eng.replay(priority=True)
        # wrong sizes, too many zones, a table over the cap: BS_E_INVAL
        assert code(eng.upload_spread, node=(zone[:-1], counts[:, :-1])) == c.BS_E_INVAL
        assert code(eng.upload_spread, pods=cls[:-1]) == c.BS_E_INVAL
        assert code(eng.upload_spread, node=(zone, counts), n_zones=65) == c.BS_E_INVAL
        n_cls = c.SPREAD_TABLE_MAX_BYTES // (((N + 31) // 32) * 32 * 4) + 1
        assert lib.bs_upload_node_spread(h, N, 3, c.ptr(zone), n_cls, c.ptr(counts)) == c.BS_E_INVAL
        # a zone id at or above n_zones: BS_E_INDEX; a count outside [0, 2^24]: BS_E_RANGE
        assert code(eng.upload_spread, node=(zone, counts), n_zones=2) == c.BS_E_INDEX
        for v in (-1, c.SPREAD_COUNT_MAX + 1):
            bad = counts.copy()
            bad[1, 3] = v
            assert code(eng.upload_spread, node=(zone, bad)) == c.BS_E_RANGE
        bad = counts.copy()
        bad[1, 3] = c.SPREAD_COUNT_MAX
        eng.upload_spread(node=(zone, bad), n_zones=64)
        # missing sides: BS_E_STATE before anything launches, only while the weight is non-zero
        eng.evaluate()
        eng.set_spread_weight(1)
        assert code(eng.evaluate) == c.BS_E_STATE    # no pod side yet
        eng.upload_spread(pods=cls)
        eng.evaluate()
        assert code(eng.upload_spread, node=(zone[:-1], counts[:, :-1])) == c.BS_E_INVAL
        assert code(eng.evaluate) == c.BS_E_STATE    # the failing call dropped the node side
        eng.upload_spread(node=(zone, counts))
        eng.evaluate()
        # a pod class at or above n_classes: BS_E_INDEX at evaluation
        big = cls.copy()
        big[4] = counts.shape[0]
        eng.upload_spread(pods=big)
        assert code(eng.evaluate) == c.BS_E_INDEX
        eng.set_spread_weight(0)
        eng.evaluate()
        eng.set_spread_weight(1)
        eng.upload_spread(pods=cls)
        # the walk refuses a non-zero weight and runs again at 0
        assert code(lambda: eng.replay(priority=True)) == c.BS_E_INVAL
        eng.set_spread_weight(0)
        eng.replay(priority=True)
    finally:
        eng.close()


def test_full_size_cfg4(pkg, oracle, snapshot_mod):
    snap = snapshot_mod.config(4)
    nz = snapshot_mod.nonzero_requests(snap, 4)
    spread = snapshot_mod.node_spread(snap, 4, n_zones=8, n_classes=32)
    eng = _engine(pkg, snap, 16, nz, spread, 1, fit_bitmap=False)
    try:
        res = eng.evaluate()
        nodes, scores = eng.priority_rows()
    finally:
        eng.close()
    idx = np.sort(np.random.default_rng(4).choice(snap.pods.n, 200, replace=False))
    want_n, want_s = sr.priority_rows(snap, nz[0], nz[1], 16, spread, 1, pods=idx)
    np.testing.assert_array_equal(nodes[idx], want_n)
    np.testing.assert_array_equal(scores[idx], want_s)
    np.testing.assert_array_equal((nodes >= 0).sum(axis=1), np.minimum(16, res.feasible_count))


def test_plugin_selector_spread_weight():
    """The C++ plugin's SetSelectorSpreadWeight(1) over objects: PriorityNodes equals an engine called directly with
    PackSpread's columns, and ReplayQueue(kPriority) refuses the weight."""
    import json
    import subprocess

    import native
    o = json.loads(subprocess.check_output([native.cpp_program("plugin_spread_priority_test"), "gpu"], text=True))
    assert o["plugin"] == o["engine"]
    assert o["replay_refused"]
    assert all(len(row) == len(o["nodes"]) for row in o["plugin"])
