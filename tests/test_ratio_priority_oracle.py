"""CPU: the two restatements of the RequestedToCapacityRatio priority (tests/ratio_priority_ref.c and
tests/pyref_ratio_priority.py) agree on every branch worked by hand, on the priority lists of random snapshots and on
the replay walk; with weight 0 the walk is bs_replay_priority's."""
import numpy as np
import pytest

import pyref_ratio_priority as pyr
import pyref_replay_priority as pyrp
import ratio_priority_ref as rr
import replay_priority_ref as rpr
from randsnap import S, random_snapshot

DEFAULT = rr.DEFAULT_SHAPE
BIN_PACK = rr.BIN_PACK
FALLING = ((0, 100), (30, 0))
STEPS = ((10, 20), (40, 90), (60, 30), (100, 70))


def both(shape, lane_weights, r, c, absent=0):
    """Ratio from both restatements; they must agree."""
    a = rr.ratio_of(shape, lane_weights, r, c, absent)
    b = pyr.ratio(shape, lane_weights, absent, dict(enumerate(r)), dict(enumerate(c)))
    assert a == b, (a, b)
    return a


def test_ceil_utilization():
    assert rr.utilization(1, 3) == pyr.utilization(1, 3) == 34     # 100 - 2*100/3 = 100 - 66: the ceiling, not 33
    assert rr.utilization(0, 3) == pyr.utilization(0, 3) == 0
    assert rr.utilization(3, 3) == pyr.utilization(3, 3) == 100
    assert both(BIN_PACK, [1, 0, 0, 0], [1, 0, 0, 0], [3, 0, 0, 0]) == 34


def test_zero_capacity_and_overcommit_give_shape_100():
    for r, c in ((0, 0), (5, 0), (-5, 0), (11, 10)):
        assert rr.utilization(r, c) == pyr.utilization(r, c) == 100
    assert both(BIN_PACK, [1, 0, 0, 0], [11, 0, 0, 0], [10, 0, 0, 0]) == 100
    assert both(DEFAULT, [1, 0, 0, 0], [0, 0, 0, 0], [0, 0, 0, 0]) == 0


def test_falling_segment_truncates_toward_zero():
    # 100 + (0 - 100) * (10 - 0) / 30 = 100 - 33 = 67: the truncation rounds toward the higher score
    assert rr.shape_at(FALLING, 10) == pyr.broken_linear(FALLING, 10) == 67
    assert both(FALLING, [1, 0, 0, 0], [1, 0, 0, 0], [10, 0, 0, 0]) == 67


@pytest.mark.parametrize("p,want", [(0, 20), (5, 20), (10, 20), (11, 22), (40, 90), (41, 87), (60, 30), (61, 31),
                                    (100, 70), (-3, 20), (150, 70)])
def test_points_below_and_above(p, want):
    assert rr.shape_at(STEPS, p) == pyr.broken_linear(STEPS, p) == want
    assert rr.shape_at(((50, 40),), p) == pyr.broken_linear(((50, 40),), p) == 40


def test_zero_score_resource_drops_out():
    # cpu at util 100 scores 100 under bin-pack; memory at util 0 scores 0 and leaves the average: 100, not 50
    assert both(BIN_PACK, [1, 1, 0, 0], [10, 0, 0, 0], [10, 10, 0, 0]) == 100
    # every resource scores 0: Ratio 0
    assert both(BIN_PACK, [1, 1, 0, 0], [0, 0, 0, 0], [10, 10, 0, 0]) == 0


def test_half_rounds_away_from_zero():
    # (50 * 1 + 51 * 1) / 2 = 50.5 -> 51 (Python's round() would give 50)
    assert both(BIN_PACK, [1, 1, 0, 0], [50, 51, 0, 0], [100, 100, 0, 0]) == 51
    assert pyr.go_round(50.5) == 51 and round(50.5) == 50
    # 3 / 2 = 1.5 -> 2; 5 / 2 = 2.5 -> 3
    assert both(BIN_PACK, [1, 1, 0, 0], [1, 2, 0, 0], [100, 100, 0, 0]) == 2
    assert both(BIN_PACK, [1, 1, 0, 0], [2, 3, 0, 0], [100, 100, 0, 0]) == 3


def test_absent_weight():
    # shape(100) = 0 (the default): the absent resources leave the average
    assert both(DEFAULT, [1, 0, 0, 0], [25, 0, 0, 0], [100, 0, 0, 0], absent=5) == 75
    # shape(100) = 100 (bin-pack): they join it at 100: (25 * 1 + 100 * 3) / 4 = 81.25 -> 81
    assert both(BIN_PACK, [1, 0, 0, 0], [25, 0, 0, 0], [100, 0, 0, 0], absent=3) == 81
    assert both(BIN_PACK, [0, 0, 0, 0], [0, 0, 0, 0], [0, 0, 0, 0], absent=3) == 100


def test_negative_values_wrap():
    big = 1 << 56
    for r, c in ((-5, 10), (-big, big), (-(1 << 62), 7), (-4, -1), (-9, -2), (-(1 << 63), -1), (-(1 << 63), -3),
                 (-3, -3), (-(1 << 60), -(1 << 56)), (0, -5), (3, -1)):
        want = pyr.utilization(r, c)
        assert rr.utilization(r, c) == want, (r, c)
    # the product wraps: (7 + 2^62) * 100 = 700 + 25 * 2^64, so it is 700 and util = 100 - 700 / 7 = 0
    assert rr.utilization(-(1 << 62), 7) == pyr.utilization(-(1 << 62), 7) == 0
    # MinInt64 / -1 is MinInt64 in Go: util = 100 - MinInt64 wraps to MinInt64 + 100
    assert rr.utilization(-(1 << 63) + 1, -1) == pyr.utilization(-(1 << 63) + 1, -1)
    for shape in (DEFAULT, BIN_PACK, FALLING, STEPS):
        both(shape, [1, 0, 1, 0, 1], [0, 0, -(1 << 60), 0, -5], [10, 10, -(1 << 56), 0, 3])


def _scalar_snapshot(seed, L=6):
    """A small snapshot whose scalar lanes are absent on some nodes and pods, with a few negative values."""
    snap = random_snapshot(seed, P=40, N=30, G=6, L=L, case="mixed")
    rng = np.random.default_rng(seed)
    nt, pt = snap.nodes, snap.pods
    nt.alloc[2] = np.where(rng.random(nt.n) < 0.1, -(1 << 20), nt.alloc[2])
    pt.req[2] = np.where(rng.random(pt.n) < 0.1, -(1 << 10), pt.req[2])
    return snap


@pytest.mark.parametrize("seed", range(4))
def test_absent_scalar_keys(seed):
    """Scalar keys present on one side only count 0 on the other; both restatements' lists agree."""
    snap = _scalar_snapshot(700 + seed)
    nz = S.nonzero_requests(snap, seed)
    lw = [1, 1, 2, 0] + [3] * (snap.lanes - 4)
    setting = (2, BIN_PACK, lw, 1)
    assert ((snap.nodes.alloc_present >> 4) & 1).min() == 0 or ((snap.pods.req_present >> 4) & 1).min() == 0
    _rows_agree(snap, nz, 8, setting, (1, 0, 1))


def _rows_agree(snap, nz, K, setting, weights):
    nodes, scores = rr.priority_rows(snap, nz[0], nz[1], K, setting, weights)
    want = pyr.priority_rows(snap, nz[0], nz[1], K, setting, weights)
    for p, row in enumerate(want):
        assert nodes[p].tolist() == [n for n, _ in row], p
        assert scores[p].tolist() == [s for _, s in row], p
    return nodes, scores


SHAPES = [DEFAULT, BIN_PACK, FALLING, STEPS, ((50, 40),), tuple((u, (u * 37) % 101) for u in range(101))]
WEIGHT_SETS = [(0, 0, 0), (1, 0, 1), (0, 1, 0), (3, 0, 7)]


@pytest.mark.parametrize("seed", range(24))
def test_random_lists_agree(seed):
    L = [4, 5, 6, 9, 12, 16][seed % 6]
    snap = random_snapshot(7000 + seed, P=30, N=[25, 40, 61][seed % 3], G=6, L=L, case=["mixed", "A", "B"][seed % 3])
    rng = np.random.default_rng(seed)
    lw = [int(x) for x in rng.integers(0, 5, L)]
    lw[3] = 0
    setting = (int(rng.integers(1, 4)), SHAPES[seed % len(SHAPES)], lw, int(rng.integers(0, 3)))
    _rows_agree(snap, S.nonzero_requests(snap, seed), 7, setting, WEIGHT_SETS[seed % 4])


def test_weight_zero_lists_are_the_priority_lists():
    import priority_ref
    snap = random_snapshot(7100, P=40, N=50, G=6, L=6, case="mixed")
    nz = S.nonzero_requests(snap, 1)
    got = rr.priority_rows(snap, nz[0], nz[1], 9, (0, BIN_PACK, [1, 1, 1, 0, 1, 1], 2))
    want = priority_ref.priority_rows(snap, nz[0], nz[1], 9)
    np.testing.assert_array_equal(got[0], want[0])
    np.testing.assert_array_equal(got[1], want[1])


AFTER = ("node_requested", "node_pod_count", "node_req_present", "group_matched", "group_flags", "group_min_res",
         "group_min_res_present", "group_rep_sel", "group_rep_tol")


@pytest.mark.parametrize("seed", range(12))
def test_replay_agrees(seed):
    L = [4, 5, 6, 9, 12, 16][seed % 6]
    snap = random_snapshot(7200 + seed, P=60, N=[30, 45][seed % 2], G=10, L=L, case=["mixed", "A", "B"][seed % 3])
    node_nz, pod_nz = S.nonzero_requests(snap, seed)
    rng = np.random.default_rng(seed)
    lw = [int(x) for x in rng.integers(0, 4, L)]
    lw[3] = 0
    setting = (int(rng.integers(1, 5)), SHAPES[seed % len(SHAPES)], lw, seed % 2)
    w = WEIGHT_SETS[seed % 4]
    queue = None if seed % 2 == 0 else rng.permutation(snap.pods.n)
    pf, node, ready, after, nz = rr.replay_ratio(snap, node_nz, pod_nz, setting, queue, w)
    ppf, pnode, pready, pafter = pyrp.replay(snap, queue, pyr.RatioChooser(node_nz, pod_nz, w, setting))
    np.testing.assert_array_equal(pf, ppf)
    np.testing.assert_array_equal(node, pnode)
    np.testing.assert_array_equal(ready, pready)
    nt, gt = after.nodes, after.groups
    got = dict(node_requested=nt.requested, node_pod_count=nt.pod_count, node_req_present=nt.req_present,
               group_matched=gt.matched, group_flags=gt.flags, group_min_res=gt.min_res,
               group_min_res_present=gt.min_res_present, group_rep_sel=gt.rep_sel, group_rep_tol=gt.rep_tol)
    for k in AFTER:
        np.testing.assert_array_equal(got[k], pafter[k], err_msg=k)
    np.testing.assert_array_equal(nz, pafter["node_nonzero"])


@pytest.mark.parametrize("seed", range(4))
def test_replay_weight_zero_is_priority_choose(seed):
    snap = random_snapshot(7300 + seed, P=80, N=50, G=10, L=[5, 6, 9, 16][seed], case="mixed")
    node_nz, pod_nz = S.nonzero_requests(snap, seed)
    w = WEIGHT_SETS[seed]
    got = rr.replay_ratio(snap, node_nz, pod_nz, (0, BIN_PACK, [1, 1, 1, 0] + [5] * (snap.lanes - 4), 1), None, w)
    want = rpr.replay_priority(snap, node_nz, pod_nz, None, w)
    for a, b in zip(got[:3], want[:3]):
        np.testing.assert_array_equal(a, b)
    np.testing.assert_array_equal(got[4], want[4])


def test_replay_bin_pack_by_gpu_lane():
    """Two nodes with 8 GPUs each (lane 4), node 1 already using 4; pods asking for 2 GPUs.  Ratio-only bin-pack by the
    GPU lane fills node 1 first (util 75 then 100), then node 0; the default spreading shape takes node 0 until it ties
    and then fills up (25 against 25 at 6 of 8), and sends the last pod to node 1."""
    L = 5
    nt = S.NodeTable.empty(2, L)
    nt.alloc[S.LANE_CPU], nt.alloc[S.LANE_MEM], nt.alloc[S.LANE_PODS], nt.alloc[4] = 64000, 256 * S.GiB, 110, 8
    nt.alloc_present[:] = 1 << 4
    nt.requested[4, 1] = 4
    nt.req_present[:] = 1 << 4   # a node fits a GPU pod only when its requested carries the key (core.go:662-666)
    pt = S.PodTable.empty(4, L)
    pt.req[S.LANE_CPU], pt.req[S.LANE_MEM], pt.req[4] = 1000, S.GiB, 2
    pt.req_present[:] = 1 << 4
    snap = S.Snapshot(nt, pt, S.GroupTable.empty(0, L), "gpu bin-pack")
    node_nz = np.zeros((2, 2), np.int64)
    pod_nz = np.array([[1000] * 4, [S.GiB] * 4], np.int64)
    pack = (1, BIN_PACK, [0, 0, 0, 0, 1], 0)
    spread = (1, DEFAULT, [0, 0, 0, 0, 1], 0)
    for setting, want in ((pack, [1, 1, 0, 0]), (spread, [0, 0, 0, 1])):
        node = rr.replay_ratio(snap, node_nz, pod_nz, setting, None, (0, 0, 0))[1]
        assert node.tolist() == want, setting
        assert pyrp.replay(snap, None, pyr.RatioChooser(node_nz, pod_nz, (0, 0, 0), setting))[1].tolist() == want
