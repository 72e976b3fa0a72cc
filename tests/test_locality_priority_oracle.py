"""CPU: the two restatements of the ImageLocality and NodePreferAvoidPods priorities (tests/locality_priority_ref.c and
tests/pyref_locality_priority.py) agree on the cases worked by hand (both thresholds, binary64 scaling, a repeated
image, a name reported outside the fit set, the controller rule), on random snapshots alone and combined with the
resource weights, the ratio term and the node priorities, and on the replay walk; with both weights 0 the lists and
the walk are the existing ones."""
import numpy as np
import pytest

import locality_priority_ref as lr
import node_priority_ref as npr
import priority_ref as pr
import pyref_locality_priority as pyl
import pyref_replay_priority as pyrp
import ratio_priority_ref as rr
import replay_priority_ref as rpr
from randsnap import S, random_snapshot

MIB = 1 << 20
NONE, ANONE = S.IMAGE_NONE, S.AVOID_NONE
LW = [(1, 0), (0, 10000), (1, 10000), (3, 7)]


def _bits(present):
    """[I, ceil(N/32)] uint32 of an [I, N] bool matrix."""
    present = np.asarray(present, bool)
    I, N = present.shape
    W = (N + 31) // 32
    pad = np.zeros((I, W * 32), bool)
    pad[:, :N] = present
    return (pad.reshape(I, W, 32).astype(np.uint64) << np.arange(32, dtype=np.uint64)).sum(
        axis=2, dtype=np.uint64).astype(np.uint32)


def _loc(sizes, present, classes, pod_class, avoid=None, abit=None):
    """Columns from a size list, an [I, N] presence matrix, class id lists and each pod's class."""
    N, P = np.asarray(present).shape[1], len(pod_class)
    off = np.concatenate([[0], np.cumsum([len(c) for c in classes])]).astype(np.uint32)
    ids = np.array([i for c in classes for i in c], np.uint32)
    avoid = np.zeros(N, np.uint64) if avoid is None else np.asarray(avoid, np.uint64)
    abit = np.full(P, ANONE, np.uint8) if abit is None else np.asarray(abit, np.uint8)
    return ((np.asarray(sizes, np.int64), _bits(present), avoid),
            (np.asarray(pod_class, np.uint32), off, ids, abit))


def _il(snap, loc, p, n):
    return int(lr.il_matrix(snap, loc, [p])[0, n])


def _py_il(loc, p, n, n_nodes):
    (size, bits, _), (cls, off, ids, _) = loc
    states = pyl.image_states(size, bits, n_nodes)
    return pyl.image_locality(states, bits, pyl.pod_ids(cls[p], off, ids), n, n_nodes)


def _agree(snap, nz, K, loc, lw, ratio=npr.NO_RATIO, weights=(1, 0, 1), prefs=None, pw=(0, 0)):
    nodes, scores = lr.priority_rows(snap, nz[0], nz[1], K, loc, lw, ratio, weights, prefs, pw)
    want = pyl.priority_rows(snap, nz[0], nz[1], K, loc, lw, ratio, weights, prefs, pw)
    for p, row in enumerate(want):
        assert nodes[p].tolist() == [n for n, _ in row], p
        assert scores[p].tolist() == [s for _, s in row], p
    return nodes, scores


def test_scaling_is_binary64():
    # 100 MiB on 29 of 100 nodes: 0.29 is below its decimal value in binary64, so the product truncates to ...703
    assert lr.image_scaled(100 * MIB, 29, 100) == 30408703 == pyl.scaled_image_score(100 * MIB, 29, 100)
    assert 100 * MIB * 29 // 100 == 30408704
    assert lr.image_scaled(500 * MIB, 1, 3) == 174762666 == pyl.scaled_image_score(500 * MIB, 1, 3)
    assert lr.image_locality(174762666) == 14 == pyl.calculate_priority(174762666)
    assert lr.image_scaled(0, 5, 9) == 0 and lr.image_scaled(1 << 48, 9, 9) == 1 << 48


def test_thresholds():
    for s, want in ((0, 0), (23 * MIB - 1, 0), (23 * MIB, 0), (23 * MIB + 10004000, 0), (23 * MIB + 10244588, 1),
                    (1000 * MIB - 1, 99), (1000 * MIB, 100), (2000 * MIB, 100), (1 << 54, 100)):
        assert lr.image_locality(s) == want == pyl.calculate_priority(s), s


def test_hand_cases_through_the_tables():
    """Each case one pod on a small snapshot: the IL of the C and Python restatements, against the number by hand."""
    snap = random_snapshot(1300, P=4, N=100, G=2, L=5)
    N = snap.nodes.n
    everywhere, half = np.ones(N, bool), np.arange(N) < N // 2
    only0 = np.arange(N) == 0
    first29 = np.arange(N) < 29
    cases = [
        # (sizes, presence rows, class ids, node, IL)
        ([0], [everywhere], [0], 0, 0),
        ([23 * MIB], [everywhere], [0], 0, 0),
        ([1000 * MIB], [everywhere], [0], 0, 100),
        ([2000 * MIB], [half], [0], 0, 100),                 # scaled to exactly 1000 MiB
        ([2000 * MIB], [half], [0], N - 1, 0),               # not reported there
        ([400 * MIB], [everywhere], [0, 0], 3, 79),          # a repeated image counts twice: 800 MiB
        ([400 * MIB], [everywhere], [0], 3, 38),
        ([1000 * MIB], [first29], [0], 0, 27),               # 1000 MiB * 0.29 rounds up to 304087040 in binary64
        ([500 * MIB, 30 * MIB], [only0, everywhere], [0, 1], 0, 1),   # 5 MiB + 30 MiB
    ]
    for sizes, rows, ids, n, want in cases:
        loc = _loc(sizes, rows, [ids], [0, NONE, 0, 0])
        assert _il(snap, loc, 0, n) == want == _py_il(loc, 0, n, N), (sizes, ids, n)
        assert _il(snap, loc, 1, n) == 0 == _py_il(loc, 1, n, N)   # BS_IMAGE_NONE
    # N = 3, NumNodes = 1: scaled 174762666, IL 14
    snap3 = random_snapshot(1301, P=2, N=3, G=1, L=5)
    loc = _loc([500 * MIB], [[True, False, False]], [[0]], [0, 0])
    assert lr.scaled(loc, 3).tolist() == [174762666]
    assert _il(snap3, loc, 0, 0) == 14 == _py_il(loc, 0, 0, 3)
    # N = 100, NumNodes = 29, 100 MiB: binary64 30408703 (exact arithmetic would give 30408704)
    loc = _loc([100 * MIB], [first29], [[0]], [0] * 4)
    assert lr.scaled(loc, N).tolist() == [30408703]


def test_name_outside_the_fit_set_counts_in_num_nodes():
    """A node no pod fits (nil / unschedulable / taint error) still reports its images: NumNodes counts it."""
    snap = random_snapshot(1302, P=30, N=40, G=5, L=5)
    bad = np.nonzero(snap.nodes.flags != 0)[0]
    assert len(bad)
    present = np.zeros((1, snap.nodes.n), bool)
    present[0, bad] = True
    present[0, 0 if bad[0] != 0 else 1] = True
    num = int(present.sum())
    loc = _loc([3000 * MIB], present, [[0]], [0] * snap.pods.n)
    assert lr.scaled(loc, snap.nodes.n).tolist() == [int(3000 * MIB * (num / snap.nodes.n))]
    nz = S.nonzero_requests(snap, 3)
    _agree(snap, nz, 12, loc, (1, 0))


def test_prefer_avoid_pods():
    snap = random_snapshot(1303, P=3, N=4, G=1, L=5)
    # node 0 lists controllers 0 and 5, node 1 controller 2, nodes 2-3 nothing
    avoid = [1 | (1 << 5), 1 << 2, 0, 0]
    loc = _loc([0], np.zeros((1, 4), bool), [[0]], [0, 0, 0], avoid, [ANONE, 5, 2])
    want = [[100, 100, 100, 100],   # no RC / RS controller
            [0, 100, 100, 100],     # controller 5: listed on node 0 only
            [100, 0, 100, 100]]     # controller 2
    assert lr.npa_matrix(snap, loc).tolist() == want
    assert [[pyl.prefer_avoid_pods(avoid[n], b) for n in range(4)] for b in (ANONE, 5, 2)] == want
    assert pyl.prefer_avoid_pods(1 << 63, 63) == 0


def test_normalized_image_name():
    for name, want in (("nginx", "nginx:latest"), ("nginx:1.17", "nginx:1.17"),
                       ("registry:5000/team/app", "registry:5000/team/app:latest"),
                       ("registry:5000/team/app:v2", "registry:5000/team/app:v2"),
                       ("gcr.io/x/y@sha256:ab", "gcr.io/x/y@sha256:ab")):
        assert pyl.normalized_image_name(name) == want


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("lw", LW)
def test_random_snapshots_agree(seed, lw):
    snap = random_snapshot(1310 + seed, P=50, N=45, G=8, L=5 + seed % 3)
    nz = S.nonzero_requests(snap, seed)
    _agree(snap, nz, 7, S.node_locality(snap, seed), lw)


@pytest.mark.parametrize("seed", range(2))
@pytest.mark.parametrize("ratio_on", [False, True])
@pytest.mark.parametrize("pref_on", [False, True])
def test_combined_with_ratio_and_node_priorities(seed, ratio_on, pref_on):
    snap = random_snapshot(1320 + seed, P=40, N=40, G=6, L=6)
    nz = S.nonzero_requests(snap, seed)
    loc = S.node_locality(snap, seed + 3)
    ratio = (3, rr.BIN_PACK, [1, 1, 0, 0, 2, 1]) if ratio_on else npr.NO_RATIO
    prefs = S.node_preferences(snap, seed) if pref_on else None
    for lw in ((1, 10000), (3, 7)):
        _agree(snap, nz, 9, loc, lw, ratio, (2, 1, 3), prefs, (1, 1))


@pytest.mark.parametrize("seed", range(3))
def test_zero_weights_give_existing_lists(seed):
    snap = random_snapshot(1330 + seed, P=50, N=40, G=6)
    nz = S.nonzero_requests(snap, seed)
    nodes, scores = _agree(snap, nz, 8, S.node_locality(snap, seed), (0, 0))
    n0, s0 = pr.priority_rows(snap, nz[0], nz[1], 8)
    assert np.array_equal(nodes, n0) and np.array_equal(scores, s0)


AFTER = ("node_requested", "node_pod_count", "node_req_present", "group_matched", "group_flags", "group_min_res",
         "group_min_res_present", "group_rep_sel", "group_rep_tol")


@pytest.mark.parametrize("seed", range(6))
def test_replay_agrees(seed):
    snap = random_snapshot(1340 + seed, P=50, N=[30, 45][seed % 2], G=10, L=[5, 6, 9][seed % 3],
                           case=["mixed", "A", "B"][seed % 3])
    node_nz, pod_nz = S.nonzero_requests(snap, seed)
    loc = S.node_locality(snap, seed, avoided=0.4)
    lw = LW[seed % 4]
    setting = (2, rr.BIN_PACK, [1, 1, 0, 0] + [1] * (snap.lanes - 4), 1) if seed % 2 else npr.NO_RATIO
    w = (1, 0, 1)
    queue = None if seed % 2 == 0 else np.random.default_rng(seed).permutation(snap.pods.n)
    pf, node, ready, after, nz = lr.replay_locality(snap, node_nz, pod_nz, loc, lw, setting, queue, w)
    chooser = pyl.LocalityChooser(node_nz, pod_nz, w, setting if len(setting[2]) == snap.lanes else
                                  (setting[0], setting[1], list(setting[2]) + [0] * (snap.lanes - len(setting[2]))),
                                  loc, lw, snap.nodes.n)
    ppf, pnode, pready, pafter = pyrp.replay(snap, queue, chooser)
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


@pytest.mark.parametrize("seed", range(3))
def test_replay_zero_weights_is_priority_walk(seed):
    snap = random_snapshot(1350 + seed, P=60, N=40, G=10, L=[5, 6, 9][seed])
    node_nz, pod_nz = S.nonzero_requests(snap, seed)
    got = lr.replay_locality(snap, node_nz, pod_nz, S.node_locality(snap, seed), (0, 0))
    want = rpr.replay_priority(snap, node_nz, pod_nz)
    for a, b in zip(got[:3], want[:3]):
        np.testing.assert_array_equal(a, b)
    np.testing.assert_array_equal(got[4], want[4])
