"""GPU: the priority lists of a round (BS_OUT_PRIORITY) bit-exact against the CPU restatement tests/priority_ref.c (fit
set from the oracle's bso_fit_eval), in every lane layout, at unaligned sizes, for several weight sets and list lengths,
beside every other output mode (whose outputs do not change), after row updates, at cfg4 size, with the error codes
of the C ABI, and through the C++ plugin's PriorityNodes."""
import importlib
import json
import os
import subprocess

import numpy as np
import pytest

import priority_ref
from randsnap import S, random_snapshot

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WEIGHTS = [(1, 0, 1), (0, 1, 0), (3, 2, 5), (0, 0, 0)]


def _sub(table, idx):
    """The compact table of rows `idx` (row updates)."""
    return type(table)(*(None if getattr(table, f) is None else
                         (getattr(table, f)[:, idx] if getattr(table, f).ndim == 2 else getattr(table, f)[idx])
                         for f in table.__dataclass_fields__))


def _fit_matrix(words, N):
    return np.unpackbits(words.view(np.uint8), axis=1, bitorder="little")[:, :N].astype(bool)


def _run(pkg, snap, K, weights=(1, 0, 1), seed=0, **kw):
    kw.setdefault("fit_bitmap", True)
    node_nz, pod_nz = S.nonzero_requests(snap, seed)
    eng = pkg.Engine(snap.lanes, 0, priority_k=K, **kw)
    try:
        eng.upload(snap)
        eng.upload_nonzero(node=node_nz, pods=pod_nz)
        eng.set_score_weights(*weights)
        res = eng.evaluate()
        rows = eng.priority_rows()
        fit = eng.fit_rows() if kw["fit_bitmap"] else None
    finally:
        eng.close()
    return res, rows, fit, node_nz, pod_nz


def _check(snap, K, weights, res, rows, fit, node_nz, pod_nz, pods=None):
    nodes, scores = rows
    want_n, want_s = priority_ref.priority_rows(snap, node_nz, pod_nz, K, weights, pods=pods)
    if pods is not None:
        nodes, scores = nodes[pods], scores[pods]
    np.testing.assert_array_equal(nodes, want_n)
    np.testing.assert_array_equal(scores, want_s)
    feas = res.feasible_count if pods is None else res.feasible_count[pods]
    np.testing.assert_array_equal((nodes >= 0).sum(axis=1), np.minimum(K, feas))
    if fit is not None and snap.nodes.n:
        m = _fit_matrix(fit, snap.nodes.n)
        if pods is not None:
            m = m[pods]
        r, c = np.nonzero(nodes >= 0)
        assert m[r, nodes[r, c]].all()


@pytest.mark.gpu
@pytest.mark.parametrize("L", range(4, 17))
@pytest.mark.parametrize("scale", ["normal", "big"])
def test_random_snapshots(pkg, oracle, L, scale):
    snap = random_snapshot(700 + L, P=300, N=700, G=40, L=L, value_scale=scale, aff=5 if L % 2 else 0)
    K = (1, 7, 32)[L % 3]
    w = WEIGHTS[L % len(WEIGHTS)]
    out = _run(pkg, snap, K, w, seed=L)
    _check(snap, K, w, *out)


@pytest.mark.gpu
@pytest.mark.parametrize("K", [1, 7, 32])
@pytest.mark.parametrize("w", WEIGHTS)
def test_weights_and_lengths(pkg, oracle, K, w):
    snap = random_snapshot(801, P=260, N=900, G=30, L=6, aff=3)
    out = _run(pkg, snap, K, w, seed=801)
    _check(snap, K, w, *out)


@pytest.mark.gpu
def test_all_wide_shape(pkg, oracle):
    """Every lane wide: memory beyond the narrow and scaled ranges on every node and pod."""
    snap = random_snapshot(7, P=200, N=600, G=30, L=9, value_scale="big")
    snap.nodes.alloc[0] = (1 << 40) + np.arange(snap.nodes.n) * 3
    snap.pods.req[0] = np.where(np.arange(snap.pods.n) % 2, (1 << 40) + 1001, 7)
    out = _run(pkg, snap, 16, (1, 1, 1), seed=7)
    _check(snap, 16, (1, 1, 1), *out)


@pytest.mark.gpu
def test_narrow_shape_with_ties(pkg, oracle):
    """Small values on every lane (the narrow layout) and many identical nodes: equal scores ordered by index."""
    snap = random_snapshot(9, P=150, N=800, G=20, L=5)
    nt = snap.nodes
    nt.alloc[0], nt.alloc[1], nt.alloc[2], nt.alloc[3] = 4000, 1 << 24, 1 << 20, 110
    nt.requested[0] = np.where(np.arange(nt.n) % 50 == 0, 3000, 1000)
    nt.requested[1], nt.requested[2] = 1 << 22, 0
    snap.pods.req[1] = np.minimum(snap.pods.req[1], 1 << 20)
    for K in (1, 32):
        out = _run(pkg, snap, K, (1, 0, 1), seed=9)
        _check(snap, K, (1, 0, 1), *out)


@pytest.mark.gpu
@pytest.mark.parametrize("N", [0, 1, 31, 33, 511, 513, 1025])
@pytest.mark.parametrize("K", [1, 7, 32])
def test_unaligned_sizes(pkg, oracle, N, K):
    snap = random_snapshot(N * 7 + K, P=70, N=max(N, 1), G=9, L=6, aff=3)
    if N == 0:
        snap.nodes = _sub(snap.nodes, np.zeros(0, np.int64))
        snap.aff_bits = None
        snap.pods.aff_class = None
        snap.groups.rep_aff = None
    res, rows, fit, node_nz, pod_nz = _run(pkg, snap, K, (1, 0, 1), seed=N)
    if N == 0:
        assert rows[0].shape == (70, K) and (rows[0] == -1).all() and (rows[1] == np.iinfo(np.int64).min).all()
        return
    _check(snap, K, (1, 0, 1), res, rows, fit, node_nz, pod_nz)


MODES = {
    "none": dict(fit_bitmap=False),
    "bitmap": dict(fit_bitmap=True),
    "score+bitmap": dict(fit_bitmap=True, score=True),
    "topk": dict(fit_bitmap=False, topk=8),
    "reasons": dict(fit_bitmap=False, reasons=True),
    "topk+bitmap+filter+reasons": dict(fit_bitmap=True, topk=8, filter=True, reasons=True),
}


def _everything(pkg, snap, K, kw, nz):
    eng = pkg.Engine(snap.lanes, 0, priority_k=K, **kw)
    try:
        eng.upload(snap)
        if K:
            eng.upload_nonzero(node=nz[0], pods=nz[1])
        res = eng.evaluate()
        out = {f: getattr(res, f) for f in ("prefilter", "feasible_count", "best_node", "best_score", "admit",
                                            "admit_bitmap", "new_denied", "order", "rank", "max_group", "max_finished")}
        if kw.get("fit_bitmap"):
            out["fit"] = eng.fit_rows()
        if kw.get("score"):
            out["score"] = eng.score_rows()
        if kw.get("topk"):
            out["topk"] = eng.topk_rows()
        if kw.get("reasons"):
            out["reasons"] = eng.reason_rows()
        if kw.get("filter"):
            out["filter"] = eng.filter_rows()
            out["filter_code"] = res.filter_code
        rows = eng.priority_rows() if K else None
    finally:
        eng.close()
    return out, rows


@pytest.mark.gpu
def test_flag_beside_every_mode(pkg, oracle):
    snap = random_snapshot(301, P=450, N=900, G=40, L=7, aff=4)
    nz = S.nonzero_requests(snap, 301)
    want = priority_ref.priority_rows(snap, nz[0], nz[1], 8)
    for name, kw in MODES.items():
        base, _ = _everything(pkg, snap, 0, kw, nz)
        with_p, rows = _everything(pkg, snap, 8, kw, nz)
        for k, v in base.items():
            if isinstance(v, tuple):
                for a, b in zip(v, with_p[k]):
                    np.testing.assert_array_equal(a, b, err_msg=f"{name}: {k}")
            else:
                np.testing.assert_array_equal(v, with_p[k], err_msg=f"{name}: {k}")
        np.testing.assert_array_equal(rows[0], want[0], err_msg=name)
        np.testing.assert_array_equal(rows[1], want[1], err_msg=name)


@pytest.mark.gpu
def test_row_updates_and_weight_changes(pkg, oracle):
    snap = random_snapshot(401, P=400, N=1200, G=40, L=8, aff=6)
    node_nz, pod_nz = S.nonzero_requests(snap, 401)
    eng = pkg.Engine(snap.lanes, 0, priority_k=16)
    try:
        eng.upload(snap)
        eng.upload_nonzero(node=node_nz, pods=pod_nz)
        res = eng.evaluate()
        _check(snap, 16, (1, 0, 1), res, eng.priority_rows(), eng.fit_rows(), node_nz, pod_nz)
        eng.set_score_weights(0, 1, 0)   # read by the next evaluation
        res = eng.evaluate()
        _check(snap, 16, (0, 1, 0), res, eng.priority_rows(), eng.fit_rows(), node_nz, pod_nz)
        rng = np.random.default_rng(401)
        nidx = np.sort(rng.choice(snap.nodes.n, 40, replace=False))
        nodes = snap.nodes.copy()
        nodes.flags[nidx[:10]] = S.NODE_UNSCHEDULABLE
        nodes.requested[0, nidx[20:30]] = 0
        nodes.alloc[1, nidx[30:]] = -nodes.alloc[1, nidx[30:]]   # negative allocatable memory
        eng.update_nodes(nidx, _sub(nodes, nidx))
        snap.nodes = nodes
        node_nz = node_nz.copy()
        node_nz[:, nidx[20:30]] = 0
        eng.upload_nonzero(node=node_nz)
        res = eng.evaluate()
        _check(snap, 16, (0, 1, 0), res, eng.priority_rows(), eng.fit_rows(), node_nz, pod_nz)
        eng.set_score_weights(3, 2, 5)
        res = eng.evaluate()
        _check(snap, 16, (3, 2, 5), res, eng.priority_rows(), eng.fit_rows(), node_nz, pod_nz)
    finally:
        eng.close()


@pytest.mark.gpu
def test_extreme_values(pkg, oracle):
    """Capacities of 0, negative allocatable, columns at 2^56 and requested beyond capacity on real fitting nodes."""
    snap = random_snapshot(451, P=200, N=500, G=20, L=5)
    nt, pt = snap.nodes, snap.pods
    rng = np.random.default_rng(451)
    nt.requested[:2] = 0
    pt.req[:2] = np.where(rng.random((2, pt.n)) < 0.5, 0, pt.req[:2])
    nt.alloc[0] = rng.choice([0, 0, 1, 1000, 1 << 30, -(1 << 40), 1 << 56], nt.n)
    nt.alloc[1] = rng.choice([0, 1, 1 << 20, -(1 << 20), -1, 1 << 56], nt.n)
    node_nz = rng.choice([0, 1, 100, 1 << 30, 1 << 56], (2, nt.n)).astype(np.int64)
    pod_nz = rng.choice([0, 100, 209715200, 1 << 56], (2, pt.n)).astype(np.int64)
    for w in WEIGHTS + [(1, 1, 1)]:
        eng = pkg.Engine(snap.lanes, 0, priority_k=32)
        try:
            eng.upload(snap)
            eng.upload_nonzero(node=node_nz, pods=pod_nz)
            eng.set_score_weights(*w)
            res = eng.evaluate()
            _check(snap, 32, w, res, eng.priority_rows(), eng.fit_rows(), node_nz, pod_nz)
            assert res.feasible_count.max() > 0
        finally:
            eng.close()


@pytest.mark.gpu
def test_full_size_cfg4(pkg, oracle, snapshot_mod):
    snap = snapshot_mod.config(4)
    node_nz, pod_nz = snapshot_mod.nonzero_requests(snap, 4)
    eng = pkg.Engine(snap.lanes, 0, fit_bitmap=False, priority_k=16)
    try:
        eng.upload(snap)
        eng.upload_nonzero(node=node_nz, pods=pod_nz)
        res = eng.evaluate()
        rows = eng.priority_rows()
    finally:
        eng.close()
    idx = np.sort(np.random.default_rng(4).choice(snap.pods.n, 300, replace=False))
    _check(snap, 16, (1, 0, 1), res, rows, None, node_nz, pod_nz, pods=idx)
    np.testing.assert_array_equal((rows[0] >= 0).sum(axis=1), np.minimum(16, res.feasible_count))


@pytest.mark.gpu
def test_errors(pkg):
    c = pkg.capi
    snap = random_snapshot(601, P=50, N=80, G=5, L=6)
    node_nz, pod_nz = S.nonzero_requests(snap, 601)

    def code(f, *a):
        with pytest.raises(c.BsError) as ei:
            f(*a)
        return ei.value.code

    eng = pkg.Engine(snap.lanes, 0)
    try:
        eng.upload(snap)
        eng.evaluate()
        eng.priority_k = 4
        assert code(eng.priority_rows) == c.BS_E_STATE   # no flag
    finally:
        eng.close()
    eng = pkg.Engine(snap.lanes, 0, priority_k=4)
    try:
        eng.upload(snap)
        assert code(eng.evaluate) == c.BS_E_STATE        # no columns
        eng.upload_nonzero(node=node_nz)
        assert code(eng.evaluate) == c.BS_E_STATE        # no pod column
        assert code(eng.priority_rows) == c.BS_E_STATE   # no round yet
        eng.upload_nonzero(pods=pod_nz)
        eng.evaluate()
        assert eng.priority_rows(10, 40)[0].shape == (40, 4)
        assert code(eng.priority_rows, 49, 2) == c.BS_E_INDEX
        # wrong counts, values out of range: the column is dropped
        assert code(eng.upload_nonzero, node_nz[:, :-1]) == c.BS_E_INVAL
        assert code(eng.evaluate) == c.BS_E_STATE
        eng.upload_nonzero(node=node_nz)
        bad = pod_nz.copy()
        bad[1, 3] = -1
        assert code(eng.upload_nonzero, None, bad) == c.BS_E_RANGE
        assert code(eng.evaluate) == c.BS_E_STATE
        bad[1, 3] = c.NONZERO_MAX + 1
        assert code(eng.upload_nonzero, None, bad) == c.BS_E_RANGE
        bad[1, 3] = c.NONZERO_MAX
        eng.upload_nonzero(pods=bad)
        eng.evaluate()
        # each table upload drops its column
        eng.upload_pods(snap.pods)
        assert code(eng.evaluate) == c.BS_E_STATE
        eng.upload_nonzero(pods=pod_nz)
        eng.evaluate()
        eng.update_nodes(np.array([3]), _sub(snap.nodes, np.array([3])))
        assert code(eng.evaluate) == c.BS_E_STATE
        eng.upload_nonzero(node=node_nz)
        eng.evaluate()
        eng.upload_nodes(snap.nodes)
        assert code(eng.evaluate) == c.BS_E_STATE
        eng.upload_nonzero(node=node_nz)
        eng.evaluate()
    finally:
        eng.close()


@pytest.mark.gpu
def test_plugin_priority_nodes(pkg, tmp_path):
    pkg.capi.load()
    src = os.path.join(ROOT, "tests", "cpp", "plugin_priority_test.cpp")
    libdir = os.path.join(ROOT, "batch-scheduler_b200")
    binary = str(tmp_path / "plugin_priority_test")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-o", binary, src, "-L" + libdir, "-lbsched",
                           "-Wl,-rpath," + libdir, "-L/usr/local/cuda/lib64", "-Wl,-rpath,/usr/local/cuda/lib64"])
    o = json.loads(subprocess.check_output([binary, "round"], text=True))
    least, most = o["begin"]
    # the min-residual rule picks node-0 (most pod slots left); LeastAllocated + Balanced picks node-1, MostAllocated
    # node-2 (scores worked by hand: DESIGN §2's formulas on cpu 8 / memory 32Gi nodes and a 500m / 1Gi pod)
    assert least["best"] == most["best"] == 0 and least["feasible"] == 3
    assert least["nodes"] == [["node-1", 82 + 96], ["node-2", 44 + 96], ["node-0", 51 + 34]]
    assert most["nodes"] == [["node-2", 54], ["node-0", 48], ["node-1", 16]]
    assert least["empty"] == most["empty"] == 0 and least["unknown"] == 0
    least, most = o["update"]
    # node-1 at 7.5 of 8 cpus: LeastAllocated 45 + Balanced 21; the pick moves to node-2
    assert least["nodes"] == [["node-2", 140], ["node-0", 85], ["node-1", 45 + 21]]
    assert most["nodes"][0] == ["node-1", (93 + 15) // 2]
    assert o["unequal_k_fails"] == 1
