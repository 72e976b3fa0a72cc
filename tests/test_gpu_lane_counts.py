"""Every lane count L = 4..16 through every kernel whose work depends on L, with the top scalar lane (and the bottom
one) deciding each outcome: the round (fit kernel, prefix scans, PreFilter), top-K, the Filter matrix, bs_cluster_check,
bs_node_left, bs_replay with and without its block cache, node row updates, and presence masks with stray bits.  Every
output is compared bit-exactly with the CPU oracle on the designed rounds of lane_cases.py.

The builds each L runs: prefix_*_kernel<MAXL> with MAXL = 4, 5, 6, 8 (L = 7, 8), 9, 12 (L = 10..12), 16 (L = 13..16);
replay_kernel<MAXL> with MAXL = 5 (L = 4, 5), 9 (L = 6..9), 16 (L = 10..16)."""
import os
import re

import numpy as np
import pytest

import lane_cases as lc
from parity import assert_round_equal
from test_gpu_replay import replay_both
from test_gpu_topk import _check_lists

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# representative classes the replay's block cache holds a checkFit bit for; with more the walk scans every block
REPLAY_MAX_CLASSES = int(re.search(r"constexpr int REPLAY_MAX_CLASSES = (\d+);", open(
    os.path.join(ROOT, "batch-scheduler_b200", "csrc", "replay.cuh")).read()).group(1))

COMBOS = lc.combos()
IDS = [f"L{L}-d{d}-{case}" for L, d, case in COMBOS]


def snapshot(L, d, case):
    return lc.lane_snapshot(L, case, d, seed=1)


def _round(pkg, snap, **kw):
    eng = pkg.Engine(snap.lanes, 0, **kw)
    try:
        eng.upload(snap)
        res = eng.evaluate()
        out = dict(res=res, shape=eng.fit_shape())
        if kw.get("fit_bitmap", True):
            out["fit"] = eng.fit_rows()
        if kw.get("score"):
            out["score"] = eng.score_rows()
        if kw.get("topk"):
            out["topk"] = eng.topk_rows()
        if kw.get("filter"):
            out["filter"] = eng.filter_rows()
    finally:
        eng.close()
    return out


def check_round(pkg, oracle, snap):
    """Score matrix, fit bitmap and every decision vector, order and rank included; returns the fit shape."""
    out = _round(pkg, snap, fit_bitmap=True, score=True)
    orc = oracle.round(snap, want_bitmap=True, want_score=True)
    assert not orc.ref_panic
    assert_round_equal(out["res"], out["fit"], out["score"], orc)
    return out["shape"], out["res"], orc


def check_filter(pkg, oracle, snap):
    out = _round(pkg, snap, fit_bitmap=False, filter=True)
    orc = oracle.round(snap, want_bitmap=False, want_filter=True)
    np.testing.assert_array_equal(out["filter"], orc.filter_bitmap)
    np.testing.assert_array_equal(out["res"].filter_code, orc.filter_code)
    np.testing.assert_array_equal(out["res"].prefilter, orc.prefilter)


def check_cluster(pkg, oracle, snap, d, stray=0):
    """bs_cluster_check and bs_node_left for both classes at both percents.  stray: extra need presence bits that no
    lane reads."""
    eng = pkg.Engine(snap.lanes)
    try:
        eng.upload_nodes(snap.nodes)
        for sel in (lc.CLS_ALL, lc.CLS_LOW):
            for pct in (1.0, 0.7):
                need, npres = lc.cluster_needs(snap, d, sel, pct)
                exp = lc.cluster_answers(oracle, snap, need, npres, sel, pct)
                got = eng.cluster_check(sel, 0, pct, need, npres | np.uint32(stray))
                bad = np.flatnonzero(got != exp)
                assert not len(bad), (sel, pct, [(need[d, j], hex(npres[j]), exp[j]) for j in bad[:4]])
                assert exp.any() and not exp.all()
                left, pres = eng.node_left(sel, 0, pct)
                el, ep = oracle.node_left(snap.nodes, sel, 0, pct)
                np.testing.assert_array_equal(left, el)
                np.testing.assert_array_equal(pres, ep)
    finally:
        eng.close()


@pytest.mark.parametrize("L,d,case", COMBOS, ids=IDS)
def test_round(pkg, oracle, L, d, case):
    snap = snapshot(L, d, case)
    shape, res, orc = check_round(pkg, oracle, snap)
    print(f"L={L} d={d} {case}: fit shape (LW, LN, LS) = ({shape['LW']}, {shape['LN']}, {shape['LS']})")
    assert sum(shape.values()) == L, shape
    if case == "B" and d >= 4:
        assert shape["LN"] == 0, shape           # no fixed lane is narrow: the all-wide fallback
    assert (orc.feasible_count > 0).any() and (orc.feasible_count < snap.nodes.n).all()


def test_fit_shapes_include_narrow_and_all_wide(pkg):
    shapes = {}
    for L, d, case in COMBOS:
        if case == "B":
            continue
        shapes[(L, d, case)] = _round(pkg, snapshot(L, d, case), fit_bitmap=True)["shape"]
    for k, s in shapes.items():
        print(k, s)
    assert any(s["LN"] > 0 for s in shapes.values()) and any(s["LN"] == 0 for s in shapes.values())
    # with ten or more lanes the narrow cap turns the top scalar lane wide (or the round goes all-wide)
    assert all(s["LN"] <= 8 for s in shapes.values())


@pytest.mark.parametrize("L,d,case", COMBOS, ids=IDS)
def test_topk(pkg, oracle, L, d, case):
    snap = snapshot(L, d, case)
    out = _round(pkg, snap, fit_bitmap=True, topk=8)
    orc = oracle.round(snap, want_bitmap=True, want_score=True)
    assert_round_equal(out["res"], out["fit"], None, orc)
    nodes, scores = out["topk"]
    _check_lists(out["res"], nodes, scores, orc.score, 8)


@pytest.mark.parametrize("L,d,case", COMBOS, ids=IDS)
def test_filter_matrix(pkg, oracle, L, d, case):
    check_filter(pkg, oracle, snapshot(L, d, case))


@pytest.mark.parametrize("L,d,case", COMBOS, ids=IDS)
def test_cluster_check_and_node_left(pkg, oracle, L, d, case):
    check_cluster(pkg, oracle, snapshot(L, d, case), d)


def _engine_order(pkg, snap):
    eng = pkg.Engine(snap.lanes, fit_bitmap=False)
    try:
        eng.upload(snap)
        return eng.evaluate().order.copy()
    finally:
        eng.close()


def rep_classes(snap):
    """The representative classes bs_replay indexes: every pod's (selector, toleration) pair and every group's
    representative pair (no affinity classes here)."""
    pods = set(zip(snap.pods.sel_mask.tolist(), snap.pods.tol_mask.tolist()))
    return len(pods | set(zip(snap.groups.rep_sel.tolist(), snap.groups.rep_tol.tolist())))


@pytest.mark.parametrize("cache", ["cached", "uncached"])
@pytest.mark.parametrize("L,d,case", COMBOS, ids=IDS)
def test_replay(pkg, oracle, L, d, case, cache):
    """The walk in the engine's order.  More than REPLAY_MAX_CLASSES representative classes (the pods' tolerations
    differ; no node has a taint, so the verdicts stay the same) turn the block cache off."""
    snap = snapshot(L, d, case)
    if cache == "uncached":
        snap.pods.tol_mask = np.random.default_rng(L).integers(0, 1 << 20, snap.pods.n).astype(np.uint64) | \
            np.uint64(0x10)
    assert (rep_classes(snap) > REPLAY_MAX_CLASSES) == (cache == "uncached"), rep_classes(snap)
    got, _ = replay_both(pkg, oracle, snap, _engine_order(pkg, snap))
    assert (got["prefilter"] != 0).any()
    if case != "mixed":       # in "mixed" only the pods that ask 0 of the lane pass PreFilter
        assert (got["node"] >= 0).sum() >= 10


def edit_deciding_lane(snap, d, seed, n=40):
    """~40 nodes get new values and presence on lane d only: (indices, compact rows, edited snapshot)."""
    rng = np.random.default_rng(seed)
    s = snap.copy()
    nt = s.nodes
    idx = np.sort(rng.choice(nt.n, n, replace=False)).astype(np.uint32)
    lvl = rng.choice(lc.LEVELS, n)
    nt.alloc[d, idx] = np.where(lvl > 2, int(nt.alloc[d].max()) + lvl, 1)
    nt.requested[d, idx] = np.where(lvl > 2, 1, 9)
    if d >= 4:
        bit = np.uint32(1 << d)
        for m in (nt.alloc_present, nt.req_present):
            m[idx] = np.where(rng.random(n) < 0.5, m[idx] | bit, m[idx] & ~bit)
    rows = type(nt)(nt.alloc[:, idx], nt.requested[:, idx], nt.pod_count[idx], nt.alloc_present[idx],
                    nt.req_present[idx], nt.label_mask[idx], nt.taint_mask[idx], nt.flags[idx])
    return idx, rows, s


@pytest.mark.parametrize("L,d,case", COMBOS, ids=IDS)
def test_row_updates_on_the_deciding_lane(pkg, oracle, L, d, case):
    """bs_update_nodes re-derives the per-lane node statistics (the lane classes) from the changed rows: the next
    round and walk equal the oracle's on the edited tables."""
    snap = snapshot(L, d, case)
    idx, rows, edited = edit_deciding_lane(snap, d, seed=L)
    eng = pkg.Engine(L, 0, fit_bitmap=True, score=True)
    try:
        eng.upload(snap)
        eng.evaluate()
        eng.update_nodes(idx, rows)
        res = eng.evaluate()
        orc = oracle.round(edited, want_bitmap=True, want_score=True)
        assert_round_equal(res, eng.fit_rows(), eng.score_rows(), orc)
        got = eng.replay(res.order)
    finally:
        eng.close()
    pf, node, ready, after = oracle.replay(edited, res.order)
    np.testing.assert_array_equal(got["prefilter"], pf)
    np.testing.assert_array_equal(got["node"], node)
    np.testing.assert_array_equal(got["ready"], ready)
    np.testing.assert_array_equal(got["node_requested"], after.nodes.requested)
    np.testing.assert_array_equal(got["node_req_present"], after.nodes.req_present)


@pytest.mark.parametrize("L,d,case", COMBOS, ids=IDS)
def test_stray_presence_bits(pkg, oracle, L, d, case):
    """Presence masks that also carry bits 0..3 and bits of lanes >= L: no lane reads them, so every output equals
    the oracle's.  An assumed pod adds only its keys of lanes 4..L-1 to the node (bs_replay's node_req_present)."""
    snap = lc.add_stray_bits(snapshot(L, d, case), seed=L)
    check_round(pkg, oracle, snap)
    check_filter(pkg, oracle, snap)
    check_cluster(pkg, oracle, snap, d, stray=(0xFFFFFFFF & ~((1 << L) - 1)) | 0xF)
    replay_both(pkg, oracle, snap, _engine_order(pkg, snap))


@pytest.mark.parametrize("L,d,case", COMBOS, ids=IDS)
def test_stray_presence_bits_fresh_groups(pkg, oracle, L, d, case):
    """Groups without MinResources take them from their first pod (fillOccupiedObj, core.go:486-493): the round's
    capture and bs_replay's keep the pod's whole presence mask above bit 3, bits of lanes >= L included, as the
    oracle does (bs_replay's group_min_res_present)."""
    snap = lc.add_stray_bits(snapshot(L, d, case), seed=L)
    gt = snap.groups
    gt.flags &= np.uint8(~lc.S.GROUP_HAS_MINRES & 0xFF)
    gt.min_res[:] = 0
    gt.min_res_present[:] = 0
    check_round(pkg, oracle, snap)
    check_filter(pkg, oracle, snap)
    got, after = replay_both(pkg, oracle, snap, _engine_order(pkg, snap))
    high = np.uint32(0xFFFFFFFF & ~((1 << L) - 1))
    assert (after.groups.min_res_present & high).any()      # the capture ran with stray bits
    assert (got["node"] >= 0).any() and ((got["node_req_present"] ^ snap.nodes.req_present) & high).sum() == 0
