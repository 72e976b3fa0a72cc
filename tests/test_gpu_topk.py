"""Top-K node lists (BS_OUT_TOPK): each pod's K best fitting nodes and their scores, without the score matrix.

The expected lists come from the CPU oracle's score matrix: a row's fitting entries ordered by score descending, then
node index ascending, cut to K and padded with node -1 / score INT64_MIN.  Every other output of a top-K round must
equal the oracle's as well.  The config checks at the top need no device."""
import json
import os
import re
import subprocess

import numpy as np
import pytest

import native
from parity import assert_round_equal
from randsnap import random_snapshot

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
I64_MIN = np.iinfo(np.int64).min


def expected_topk(score, K):
    """[P, N] oracle scores (INT64_MIN = does not fit) -> (nodes [P, K] int32, scores [P, K] int64)."""
    P, N = score.shape
    nodes = np.full((P, K), -1, np.int32)
    scores = np.full((P, K), I64_MIN, np.int64)
    if N == 0:
        return nodes, scores
    fit = score != I64_MIN
    key = np.where(fit, score, -1)                     # fitting scores are >= 0
    idx = np.broadcast_to(np.arange(N), (P, N))
    order = np.lexsort((idx, -key), axis=1)[:, :K]     # score descending, then node ascending
    take = min(K, N)
    ok = np.take_along_axis(fit, order, axis=1)
    nodes[:, :take] = np.where(ok, order, -1)
    scores[:, :take] = np.where(ok, np.take_along_axis(score, order, axis=1), I64_MIN)
    return nodes, scores


# ---- CPU: the config contract, checked before the device probe ------------------------------------------------

def _create(pkg, flags, k, lanes=5):
    capi = pkg.capi
    lib = capi.load()
    import ctypes as C
    h = C.c_void_p()
    rc = lib.bs_create(C.byref(capi.Config(0, lanes, flags, k)), C.byref(h))
    if rc == 0:
        lib.bs_destroy(h)
    return rc


def test_topk_constants_agree(pkg):
    hdr = open(os.path.join(ROOT, "include", "bsched.h")).read()
    assert int(re.search(r"#define BS_OUT_TOPK (0x[0-9a-fA-F]+)u", hdr).group(1), 16) == pkg.capi.OUT_TOPK == 0x8
    assert int(re.search(r"#define BS_TOPK_MAX (\d+)", hdr).group(1)) == pkg.capi.TOPK_MAX == 32
    assert "bs_fetch_topk_rows" in pkg.capi.SYMBOLS and hasattr(pkg.capi.load(), "bs_fetch_topk_rows")
    assert [f[0] for f in pkg.capi.Config._fields_] == ["device", "n_lanes", "out_flags", "topk"]


@pytest.mark.parametrize("flags,k", [
    ("topk", 0),            # the flag needs a list length
    ("topk", 33),           # longer than BS_TOPK_MAX
    ("bitmap", 4),          # a list length without the flag
    ("topk|score", 8),      # the score matrix already holds every list
])
def test_topk_config_rejected(pkg, flags, k):
    c = pkg.capi
    f = {"topk": c.OUT_TOPK, "bitmap": c.OUT_FIT_BITMAP, "topk|score": c.OUT_TOPK | c.OUT_SCORE}[flags]
    assert _create(pkg, f, k) == c.BS_E_INVAL


def test_topk_config_accepted(pkg):
    import torch
    c = pkg.capi
    want = c.BS_OK if torch.cuda.is_available() else c.BS_E_NODEVICE
    for f, k in ((c.OUT_TOPK, 1), (c.OUT_TOPK | c.OUT_FIT_BITMAP | c.OUT_FILTER, 32), (c.OUT_FIT_BITMAP, 0)):
        assert _create(pkg, f, k) == want, (f, k)


# ---- GPU -------------------------------------------------------------------------------------------------------

def _round(pkg, snap, K, bitmap):
    eng = pkg.Engine(snap.lanes, 0, fit_bitmap=bitmap, topk=K)
    try:
        eng.upload(snap)
        res = eng.evaluate()
        fit = eng.fit_rows() if bitmap else None
        nodes, scores = eng.topk_rows()
    finally:
        eng.close()
    return res, fit, nodes, scores


def _check_lists(res, nodes, scores, score_matrix, K):
    en, es = expected_topk(score_matrix, K)
    np.testing.assert_array_equal(nodes, en, err_msg="top-K nodes")
    np.testing.assert_array_equal(scores, es, err_msg="top-K scores")
    np.testing.assert_array_equal(nodes[:, 0], res.best_node, err_msg="entry 0 = best_node")
    np.testing.assert_array_equal(scores[:, 0], res.best_score, err_msg="entry 0 = best_score")
    np.testing.assert_array_equal((nodes >= 0).sum(axis=1), np.minimum(K, res.feasible_count))


def _run(pkg, oracle, snap, K, bitmap=False):
    res, fit, nodes, scores = _round(pkg, snap, K, bitmap)
    orc = oracle.round(snap, want_bitmap=True, want_score=True)
    assert not orc.ref_panic
    assert nodes.shape == scores.shape == (snap.pods.n, K)
    assert_round_equal(res, fit, None, orc)
    _check_lists(res, nodes, scores, orc.score, K)
    return res, nodes, scores


@pytest.mark.gpu
@pytest.mark.parametrize("K", [1, 5, 16, 32])
@pytest.mark.parametrize("bitmap", [True, False])
@pytest.mark.parametrize("seed,kw", [(11, {}), (12, {"value_scale": "big"}), (13, {"aff": 6}), (14, {"case": "B"})])
def test_topk_random_parity(pkg, oracle, K, bitmap, seed, kw):
    _run(pkg, oracle, random_snapshot(seed, P=700, N=1100, G=60, **kw), K, bitmap)


def _mixed(seed, P, N):
    # lane 0 (cpu) narrow, lane 1 (odd memory values above 2^27) wide, lane 2 (multiples of 2^20) scaled
    snap = random_snapshot(seed, P=P, N=N, G=40, L=6)
    nt, pt = snap.nodes, snap.pods
    rng = np.random.default_rng(seed)
    nt.alloc[0] = rng.integers(1000, 64000, N)
    nt.requested[0] = rng.integers(0, 32000, N)
    pt.req[0] = rng.choice([0, 100, 500, 2000, 8000], P)
    nt.alloc[2] = rng.integers(1, 1 << 12, N) << 20
    nt.requested[2] = rng.integers(0, 1 << 11, N) << 20
    pt.req[2] = rng.integers(0, 1 << 10, P) << 20
    return snap


def _all_wide(seed, P, N):
    snap = random_snapshot(seed, P=P, N=N, G=40, L=5)
    nt, pt = snap.nodes, snap.pods
    rng = np.random.default_rng(seed)
    for d in range(5):
        nt.alloc[d] = rng.integers(1 << 30, 1 << 45, N)
        pt.req[d] = rng.integers(0, 1 << 44, P)
    return snap


# odd N, a partial last tile, P not a multiple of 32, and a partial last wave (which top-K mode does not split)
SHAPES = [(3001, 3001), (2999, 2050), (1000, 4097)]


@pytest.mark.gpu
@pytest.mark.parametrize("P,N", SHAPES)
@pytest.mark.parametrize("layout", ["mixed", "all_wide"])
def test_topk_lane_shapes(pkg, oracle, P, N, layout):
    gen = _mixed if layout == "mixed" else _all_wide
    snap = gen(9000 + P + N, P, N)
    eng = pkg.Engine(snap.lanes, 0, fit_bitmap=False, topk=16)
    eng.upload(snap)
    eng.evaluate()
    shape = eng.fit_shape()
    eng.close()
    assert (shape["LN"] == 0) == (layout == "all_wide"), shape
    _run(pkg, oracle, snap, 16, bitmap=(P == 2999))


def _plain(seed, P, N, L=5):
    """A snapshot whose only limits are the resource lanes: no flags, masks, taints or deny state."""
    snap = random_snapshot(seed, P=P, N=N, G=20, L=L)
    nt, pt = snap.nodes, snap.pods
    nt.flags[:] = 0
    nt.label_mask[:] = 0
    nt.taint_mask[:] = 0
    pt.sel_mask[:] = 0
    pt.tol_mask[:] = 0
    return snap


@pytest.mark.gpu
@pytest.mark.parametrize("N", [0, 1, 7])
def test_topk_fewer_nodes_than_k(pkg, oracle, N):
    _, nodes, _ = _run(pkg, oracle, random_snapshot(21 + N, P=90, N=N, G=8, L=5), 16)
    assert (nodes[:, max(N, 0):] == -1).all()


@pytest.mark.gpu
def test_topk_pods_that_fit_nowhere(pkg, oracle):
    snap = _plain(31, 200, 1500)
    snap.pods.req[0, ::3] = 1 << 40                     # more cpu than any node has
    res, nodes, scores = _run(pkg, oracle, snap, 8)
    assert (res.feasible_count[::3] == 0).all()
    assert (nodes[::3] == -1).all() and (scores[::3] == I64_MIN).all()


@pytest.mark.gpu
@pytest.mark.parametrize("K", [5, 32])
def test_topk_equal_scores_tie_on_node_index(pkg, oracle, K):
    # five distinct node rows repeated over 2000 nodes: long runs of equal scores, ordered by node index
    snap = _plain(41, 300, 2000)
    nt = snap.nodes
    proto = np.arange(2000) % 5
    for d in range(nt.lanes):
        nt.alloc[d] = nt.alloc[d][proto]
        nt.requested[d] = nt.requested[d][proto]
    nt.pod_count = nt.pod_count[proto]
    nt.alloc_present = nt.alloc_present[proto]
    nt.req_present = nt.req_present[proto]
    _, nodes, scores = _run(pkg, oracle, snap, K)
    full = (nodes >= 0).all(axis=1)
    assert full.any() and (np.diff(scores[full], axis=1) == 0).any()


@pytest.mark.gpu
@pytest.mark.parametrize("direction", ["rising", "falling"])
def test_topk_monotone_residuals(pkg, oracle, direction):
    # free cpu rising with node index: every fitting node enters the list; falling: none after the first K
    P, N = 500, 3000
    snap = _plain(51, P, N, L=4)
    nt, pt = snap.nodes, snap.pods
    free = np.arange(N, dtype=np.int64) * 7 + 9000
    if direction == "falling":
        free = free[::-1].copy()
    nt.alloc[0] = 64000 + free
    nt.requested[0] = 64000
    for d in range(1, 4):
        nt.alloc[d] = 1 << 40
        nt.requested[d] = 0
    pt.req[0] = np.random.default_rng(51).integers(0, 8000, P)
    for d in range(1, 4):
        pt.req[d] = 0
    _, nodes, _ = _run(pkg, oracle, snap, 16)
    lead = nodes[:, 0][nodes[:, 0] >= 0]
    assert (lead == (N - 1 if direction == "rising" else 0)).all()


@pytest.mark.gpu
def test_topk_row_updates(pkg, oracle):
    snap = random_snapshot(61, P=600, N=1300, G=50, L=6)
    eng = pkg.Engine(snap.lanes, 0, fit_bitmap=False, topk=12)
    try:
        eng.upload(snap)
        eng.evaluate()
        rng = np.random.default_rng(61)
        nidx = np.sort(rng.choice(snap.nodes.n, 9, replace=False))
        rows = snap.nodes.copy()
        for d in range(3):
            rows.requested[d, nidx] = 0                  # the changed nodes free up
        rows.flags[nidx[:2]] = 0
        eng.update_nodes(nidx, rows.take(nidx))
        snap.nodes = rows
        gidx = np.sort(rng.choice(snap.groups.n, 5, replace=False))
        groups = snap.groups.copy()
        groups.matched[gidx] += 1
        groups.flags[gidx] ^= 0x8                          # toggles GROUP_DENIED
        eng.update_groups(gidx, groups.take(gidx))
        snap.groups = groups
        res = eng.evaluate()
        nodes, scores = eng.topk_rows()
    finally:
        eng.close()
    orc = oracle.round(snap, want_bitmap=False, want_score=True)
    assert_round_equal(res, None, None, orc)
    _check_lists(res, nodes, scores, orc.score, 12)


@pytest.mark.gpu
def test_topk_group_shards(pkg, oracle):
    full = random_snapshot(71, P=1200, N=900, G=80, L=6).resolve_groups()
    for r in range(2):
        snap = full.shard_groups(r, 2)
        res, fit, nodes, scores = _round(pkg, snap, 10, False)
        orc = oracle.round(snap, want_bitmap=False, want_score=True)
        _check_lists(res, nodes, scores, orc.score, 10)


@pytest.mark.gpu
def test_topk_full_size_cfg4(pkg, oracle, snapshot_mod):
    S = snapshot_mod
    snap = S.config(4)
    eng = pkg.Engine(snap.lanes, 0, fit_bitmap=False, topk=16)
    eng.upload(snap)
    res = eng.evaluate()
    idx = np.sort(np.random.default_rng(4).choice(snap.pods.n, 300, replace=False))
    nodes, scores = eng.topk_rows()
    eng.close()
    sub = S.Snapshot(snap.nodes, snap.pods.take(idx), snap.groups)
    o2 = oracle.round(sub, want_bitmap=False, want_score=True, want_sort=False, threads=0)
    en, es = expected_topk(o2.score, 16)
    np.testing.assert_array_equal(nodes[idx], en)
    np.testing.assert_array_equal(scores[idx], es)
    np.testing.assert_array_equal(nodes[:, 0], res.best_node)
    np.testing.assert_array_equal(scores[:, 0], res.best_score)
    np.testing.assert_array_equal((nodes >= 0).sum(axis=1), np.minimum(16, res.feasible_count))


@pytest.mark.gpu
def test_plugin_top_nodes():
    K = 8
    rounds = json.loads(subprocess.check_output([native.cpp_program("plugin_topk_test"), "topk", str(K)], text=True))
    assert len(rounds) == 2                            # BeginRound, then UpdateRound
    for rd in rounds:
        assert rd["rc"] == 0 and rd["unknown"] == 0
        rn = np.array(rd["rows_node"]).reshape(-1, K)
        rs = np.array(rd["rows_score"]).reshape(-1, K)
        feas = np.array(rd["feasible"])
        assert (rn[:, 0] == np.array(rd["best"])).all()
        for p, top in enumerate(rd["top"]):
            want = [[f"node-{n}", int(s)] for n, s in zip(rn[p], rs[p]) if n >= 0]
            assert top == want, p
            assert len(top) == min(K, feas[p])
        assert rd["top"][7] == []                       # fits nowhere
    before, after = (np.array(rd["rows_node"]).reshape(-1, K) for rd in rounds)
    assert (after == 5).any() and not (before == 5).any()     # an emptied node enters the lists ...
    assert (after == 280).sum() < (before == 280).sum()        # ... ahead of a later node of equal score
    assert not (after == 150).any()                            # a full node fits nowhere
