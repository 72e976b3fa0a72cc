"""GPU: the TaintToleration and preferred NodeAffinity priorities (bs_set_node_priority_weights) in the round's priority
lists, bit-exact against the CPU restatement tests/node_priority_ref.c: every lane build, list lengths, unaligned sizes,
four weight pairs, with the ratio term on and off; weights (0, 0) are the engine without them; the other outputs do not
move; the node side follows bs_update_nodes; every error code; sampled pods at cfg4 size; and the C++ plugin's
SetNodePriorityWeights over objects with soft taints and preferred terms."""
import json
import subprocess

import numpy as np
import pytest

import native
import node_priority_ref as npr
import ratio_priority_ref as rr
from randsnap import S, random_snapshot

pytestmark = pytest.mark.gpu

PW = [(1, 0), (0, 1), (1, 1), (3, 7)]


def _ratio(L, on):
    return (2, rr.BIN_PACK, [1, 1, 0, 0] + [1] * (L - 4), 1) if on else npr.NO_RATIO


def _engine(pkg, snap, K, nz, prefs, pw, ratio=None, weights=(1, 0, 1), **kw):
    eng = pkg.Engine(snap.lanes, 0, priority_k=K, **kw)
    eng.upload(snap)
    eng.upload_nonzero(node=nz[0], pods=nz[1])
    eng.set_score_weights(*weights)
    if ratio is not None and ratio[0]:
        eng.set_ratio_priority(*ratio)
    if prefs is not None:
        eng.upload_preferences(node=(prefs[0], prefs[1]), pods=(prefs[2], prefs[3]))
    eng.set_node_priority_weights(*pw)
    return eng


def _check(pkg, snap, K, pw, ratio_on, seed, weights=(1, 0, 1), prefs=None):
    nz = S.nonzero_requests(snap, seed)
    prefs = S.node_preferences(snap, seed) if prefs is None else prefs
    ratio = _ratio(snap.lanes, ratio_on)
    eng = _engine(pkg, snap, K, nz, prefs, pw, ratio, weights)
    try:
        eng.evaluate()
        nodes, scores = eng.priority_rows()
    finally:
        eng.close()
    want_n, want_s = npr.priority_rows(snap, nz[0], nz[1], K, prefs, pw, ratio, weights)
    np.testing.assert_array_equal(nodes, want_n)
    np.testing.assert_array_equal(scores, want_s)
    return nodes, scores


@pytest.mark.parametrize("L", [5, 9, 16])
@pytest.mark.parametrize("pw", PW)
@pytest.mark.parametrize("ratio_on", [False, True])
def test_lane_builds(pkg, oracle, L, pw, ratio_on):
    snap = random_snapshot(1100 + L, P=260, N=700, G=30, L=L, case="mixed")
    K = {5: 1, 9: 7, 16: 32}[L]
    _check(pkg, snap, K, pw, ratio_on, seed=L)


@pytest.mark.parametrize("K", [1, 7, 32])
@pytest.mark.parametrize("pw", PW)
def test_lengths_and_weights(pkg, oracle, K, pw):
    snap = random_snapshot(1150 + K, P=300, N=900, G=30, L=6, aff=3)
    _check(pkg, snap, K, pw, K == 7, seed=K, weights=(2, 1, 3))


@pytest.mark.parametrize("P,N", [(1, 1), (37, 31), (70, 33), (131, 511), (95, 1025)])
def test_unaligned_sizes(pkg, oracle, P, N):
    snap = random_snapshot(P * 7 + N, P=P, N=N, G=9, L=6)
    _check(pkg, snap, 7, (1, 1), N % 2 == 1, seed=N)


def test_non_fitting_node_does_not_count(pkg, oracle):
    """Every pod's weights peak on nodes it does not fit: the lists still equal the restatement over the fit set."""
    snap = random_snapshot(1190, P=200, N=400, G=20, L=6)
    taints, table, tol, cls = S.node_preferences(snap, 5, n_bits=8, tolerate=0.1, tolerate_all=0.0)
    bad = np.nonzero(snap.nodes.flags != 0)[0]   # nil / unschedulable / taint-error nodes fit no pod
    assert len(bad)
    taints[bad] = np.uint64(0xFF)
    table[:, bad] = 1 << 30
    _check(pkg, snap, 16, (1, 1), False, seed=5, prefs=(taints, table, tol, cls))
    _check(pkg, snap, 16, (3, 7), True, seed=5, prefs=(taints, table, tol, cls))


def test_zero_weights_are_the_engine_without_them(pkg, oracle):
    snap = random_snapshot(1191, P=300, N=800, G=30, L=6, aff=2)
    nz = S.nonzero_requests(snap, 1191)
    prefs = S.node_preferences(snap, 1191)
    out = []
    for with_cols in (False, True):
        eng = _engine(pkg, snap, 9, nz, prefs if with_cols else None, (0, 0))
        try:
            eng.evaluate()
            out.append(eng.priority_rows())
            if with_cols:   # on, then off again on the same engine
                eng.set_node_priority_weights(1, 1)
                eng.evaluate()
                on = eng.priority_rows()
                eng.set_node_priority_weights(0, 0)
                eng.evaluate()
                out.append(eng.priority_rows())
        finally:
            eng.close()
    for nodes, scores in out[1:]:
        np.testing.assert_array_equal(nodes, out[0][0])
        np.testing.assert_array_equal(scores, out[0][1])
    assert not np.array_equal(on[1], out[0][1])


def test_other_outputs_do_not_move(pkg, oracle):
    snap = random_snapshot(1192, P=300, N=800, G=30, L=6)
    nz = S.nonzero_requests(snap, 1192)
    prefs = S.node_preferences(snap, 1192)
    got = []
    for pw in ((0, 0), (3, 7)):
        eng = _engine(pkg, snap, 8, nz, prefs, pw, fit_bitmap=True, topk=8, reasons=True)
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


def test_node_side_follows_row_updates(pkg, oracle):
    c = pkg.capi
    snap = random_snapshot(1193, P=200, N=500, G=20, L=6)
    nz = S.nonzero_requests(snap, 1193)
    prefs = S.node_preferences(snap, 1193)
    eng = _engine(pkg, snap, 16, nz, prefs, (1, 1))
    try:
        eng.evaluate()
        idx = np.arange(0, snap.nodes.n, 7)
        rows = snap.nodes.take(idx)
        rows.label_mask = rows.label_mask ^ np.uint64(1)
        eng.update_nodes(idx, rows)
        snap2 = snap.copy()
        snap2.nodes.label_mask[idx] = rows.label_mask
        eng.upload_nonzero(node=nz[0])
        with pytest.raises(c.BsError) as ei:
            eng.evaluate()
        assert ei.value.code == c.BS_E_STATE
        taints, table = prefs[0].copy(), prefs[1].copy()
        taints[idx] = ~taints[idx] & np.uint64(0x3F)
        table[:, idx] = table[:, idx][:, ::-1]
        eng.upload_preferences(node=(taints, table))
        eng.evaluate()
        nodes, scores = eng.priority_rows()
    finally:
        eng.close()
    prefs2 = (taints, table, prefs[2], prefs[3])
    want_n, want_s = npr.priority_rows(snap2, nz[0], nz[1], 16, prefs2, (1, 1))
    np.testing.assert_array_equal(nodes, want_n)
    np.testing.assert_array_equal(scores, want_s)


def test_errors(pkg):
    c = pkg.capi
    snap = random_snapshot(1194, P=50, N=80, G=5, L=6)
    nz = S.nonzero_requests(snap, 1194)
    taints, table, tol, cls = S.node_preferences(snap, 1194)
    lib = c.load()

    def code(f, *a):
        with pytest.raises(c.BsError) as ei:
            f(*a)
        return ei.value.code

    eng = _engine(pkg, snap, 4, nz, None, (0, 0))
    try:
        # wrong sizes, negative weights, a table above the cap
        assert code(eng.upload_preferences, (taints[:-1], table[:, :-1]), None) == c.BS_E_INVAL
        assert code(eng.upload_preferences, None, (tol[:-1], cls[:-1])) == c.BS_E_INVAL
        neg = table.copy()
        neg[0, 3] = -1
        assert code(eng.upload_preferences, (taints, neg), None) == c.BS_E_RANGE
        h = eng.h
        big = c.PREF_TABLE_MAX_BYTES // (((snap.nodes.n + 31) // 32) * 32 * 4) + 1
        assert lib.bs_upload_node_preferences(h, snap.nodes.n, c.ptr(taints), big, None) == c.BS_E_INVAL
        # missing columns: BS_E_STATE before anything launches, per weight
        eng.set_node_priority_weights(1, 0)
        assert code(eng.evaluate) == c.BS_E_STATE
        eng.upload_preferences(pods=(tol, cls))
        assert code(eng.evaluate) == c.BS_E_STATE    # the node side failed above: still missing
        eng.upload_preferences(node=(taints, table))
        eng.evaluate()
        eng.upload(snap)                             # new pods and nodes drop both sides
        eng.upload_nonzero(node=nz[0], pods=nz[1])
        assert code(eng.evaluate) == c.BS_E_STATE
        eng.set_node_priority_weights(0, 1)
        eng.upload_preferences(node=(taints, table), pods=(tol, cls))
        eng.evaluate()
        # a class outside the table: BS_E_INDEX at evaluation (only where the affinity weight reads it)
        bad = cls.copy()
        bad[5] = table.shape[0]
        eng.upload_preferences(pods=(tol, bad))
        assert code(eng.evaluate) == c.BS_E_INDEX
        eng.set_node_priority_weights(1, 0)
        eng.evaluate()
        # bs_replay_priority refuses to run while either weight is non-zero, and runs again at (0, 0)
        assert code(eng.replay, None, True, True) == c.BS_E_INVAL
        assert "TaintToleration" in lib.bs_last_error(h).decode()
        eng.set_node_priority_weights(0, 0)
        eng.replay(None, True, True)
    finally:
        eng.close()


def test_full_size_cfg4(pkg, oracle, snapshot_mod):
    snap = snapshot_mod.config(4)
    nz = snapshot_mod.nonzero_requests(snap, 4)
    prefs = snapshot_mod.node_preferences(snap, 4)
    eng = _engine(pkg, snap, 16, nz, prefs, (1, 1), fit_bitmap=False)
    try:
        res = eng.evaluate()
        nodes, scores = eng.priority_rows()
    finally:
        eng.close()
    idx = np.sort(np.random.default_rng(4).choice(snap.pods.n, 200, replace=False))
    want_n, want_s = npr.priority_rows(snap, nz[0], nz[1], 16, prefs, (1, 1), pods=idx)
    np.testing.assert_array_equal(nodes[idx], want_n)
    np.testing.assert_array_equal(scores[idx], want_s)
    np.testing.assert_array_equal((nodes >= 0).sum(axis=1), np.minimum(16, res.feasible_count))


def _expected_plugin_lists(o):
    """Per pod, the plugin's scenario evaluated here: the fit set (every NoSchedule / NoExecute taint tolerated), the
    raw counts from the packed columns, and the normalized sum; the resource part is the same on every node."""
    import test_plugin_node_priority as tp
    out = []
    for p, pod in enumerate(o["pods"]):
        fit = [i for i, nd in enumerate(o["nodes"])
               if all(any(tp.tolerates(t, tuple(x)) for t in pod["tolerations"])
                      for x in nd["taints"] if x[2] in ("NoSchedule", "NoExecute"))]
        t = {i: bin(o["prefer_taints"][i] & ~o["prefer_tol"][p]).count("1") for i in fit}
        cls = o["pref_class"][p]
        a = {i: 0 if cls == 0xFFFFFFFF else o["pref_weights"][cls][i] for i in fit}
        mt, ma = max(t.values(), default=0), max(a.values(), default=0)
        out.append({i: (100 if mt == 0 else 100 - 100 * t[i] // mt) + (0 if ma == 0 else 100 * a[i] // ma) for i in fit})
    return out


def test_plugin_node_priorities():
    o = json.loads(subprocess.check_output([native.cpp_program("plugin_node_priority_test"), "gpu"], text=True))
    assert o["plugin"] == o["engine"]
    assert o["replay_refused"] == 1
    names = [f"node-{i}" for i in range(len(o["nodes"]))]
    for p, (row, want) in enumerate(zip(o["plugin"], _expected_plugin_lists(o))):
        assert sorted(names.index(n) for n, _ in row) == sorted(want), p
        base = {row[0][1] - want[names.index(row[0][0])]}
        for n, s in row:
            base.add(s - want[names.index(n)])
        assert len(base) == 1, (p, row, want)   # the lists differ from the raw sums by the shared resource score
    # node-2 (NoSchedule k3) fits only pod 3, node-5 (NoExecute k5) only pods 2 and 8
    assert "node-2" in [n for n, _ in o["plugin"][3]] and "node-2" not in [n for n, _ in o["plugin"][0]]
