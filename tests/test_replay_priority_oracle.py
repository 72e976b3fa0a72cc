"""CPU: the two restatements of bs_replay_priority (tests/replay_priority_ref.c and tests/pyref_replay_priority.py)
agree with each other per queue position and on the whole after-state, the hooked walk with the first-fit chooser is
the oracle's bso_replay, weights (0, 0, 0) give first-fit exactly, and placements worked by hand."""
import numpy as np
import pytest

import pyref_replay_priority as pyr
import replay_priority_ref as rpr
from randsnap import S, random_snapshot

WEIGHTS = [(1, 0, 1), (0, 1, 0), (1, 1, 1), (3, 0, 7)]
AFTER = ("node_requested", "node_pod_count", "node_req_present", "group_matched", "group_flags", "group_min_res",
         "group_min_res_present", "group_rep_sel", "group_rep_tol")


def _after_of(s):
    """bs_replay_result's after-state fields of a walked snapshot copy."""
    nt, gt = s.nodes, s.groups
    return dict(node_requested=nt.requested, node_pod_count=nt.pod_count, node_req_present=nt.req_present,
                group_matched=gt.matched, group_flags=gt.flags, group_min_res=gt.min_res,
                group_min_res_present=gt.min_res_present, group_rep_sel=gt.rep_sel, group_rep_tol=gt.rep_tol)


def _assert_same(a, b):
    for k in AFTER:
        np.testing.assert_array_equal(a[k], b[k], err_msg=k)


@pytest.mark.parametrize("seed", range(24))
def test_c_and_python_agree(seed):
    L = [4, 5, 6, 9, 12, 16][seed % 6]
    w = WEIGHTS[seed % 4]
    snap = random_snapshot(5000 + seed, P=70, N=[30, 45, 61][seed % 3], G=10, L=L, case=["mixed", "A", "B"][seed % 3])
    node_nz, pod_nz = S.nonzero_requests(snap, seed)
    queue = None if seed % 2 == 0 else np.random.default_rng(seed).permutation(snap.pods.n)
    pf, node, ready, after, nz = rpr.replay_priority(snap, node_nz, pod_nz, queue, w)
    ppf, pnode, pready, pafter = pyr.replay(snap, queue, pyr.PriorityChooser(node_nz, pod_nz, w))
    np.testing.assert_array_equal(pf, ppf)
    np.testing.assert_array_equal(node, pnode)
    np.testing.assert_array_equal(ready, pready)
    _assert_same(_after_of(after), pafter)
    np.testing.assert_array_equal(nz, pafter["node_nonzero"])
    # the live column grew by exactly the assumed pods' columns
    want = np.asarray(node_nz, np.int64).copy()
    placed = node >= 0
    q = np.arange(snap.pods.n) if queue is None else np.asarray(queue)
    for r in range(2):
        np.add.at(want[r], node[placed], np.asarray(pod_nz)[r, q[placed]])
    np.testing.assert_array_equal(nz, want)


@pytest.mark.parametrize("seed", range(8))
def test_first_fit_hook_is_the_oracle_walk(oracle, seed):
    """The restated walk with the first-fit chooser is bso_replay, affinity classes included; so is the Python walk
    on a snapshot without them."""
    snap = random_snapshot(5100 + seed, P=120, N=80, G=14, L=[4, 6, 9, 16][seed % 4], aff=3 * (seed % 2))
    queue = None if seed % 3 else np.random.default_rng(seed).permutation(snap.pods.n)
    want = oracle.replay(snap, queue)
    got = rpr.replay_first_fit(snap, queue)
    for a, b in zip(got[:3], want[:3]):
        np.testing.assert_array_equal(a, b)
    _assert_same(_after_of(got[3]), _after_of(want[3]))
    if seed % 2 == 0:
        ppf, pnode, pready, pafter = pyr.replay(snap, queue)
        np.testing.assert_array_equal(ppf, want[0])
        np.testing.assert_array_equal(pnode, want[1])
        np.testing.assert_array_equal(pready, want[2])
        _assert_same(pafter, _after_of(want[3]))


@pytest.mark.parametrize("seed", range(6))
def test_zero_weights_are_first_fit(oracle, seed):
    """Every fitting node scores 0: the tie rule picks the lowest index, bso_replay's choice."""
    snap = random_snapshot(5200 + seed, P=150, N=90, G=16, L=[5, 6, 9][seed % 3], aff=2 * (seed % 2))
    node_nz, pod_nz = S.nonzero_requests(snap, seed)
    pf, node, ready, after, _ = rpr.replay_priority(snap, node_nz, pod_nz, None, (0, 0, 0))
    want = oracle.replay(snap)
    for a, b in zip((pf, node, ready), want[:3]):
        np.testing.assert_array_equal(a, b)
    _assert_same(_after_of(after), _after_of(want[3]))


def _two_nodes(n_pods, node0_cpu=0):
    """Two empty nodes of 4000 m / 8 GiB (node 0 at node0_cpu millicores requested), pods of 500 m / 1 GiB outside
    any group, and their non-zero columns (the requests themselves)."""
    L = 4
    nt = S.NodeTable.empty(2, L)
    nt.alloc[S.LANE_CPU], nt.alloc[S.LANE_MEM], nt.alloc[S.LANE_PODS] = 4000, 8 * S.GiB, 110
    nt.requested[S.LANE_CPU, 0] = node0_cpu
    pt = S.PodTable.empty(n_pods, L)
    pt.req[S.LANE_CPU], pt.req[S.LANE_MEM] = 500, S.GiB
    snap = S.Snapshot(nt, pt, S.GroupTable.empty(0, L), "two nodes")
    node_nz = np.array([[node0_cpu, 0], [0, 0]], np.int64)
    pod_nz = np.array([[500] * n_pods, [S.GiB] * n_pods], np.int64)
    return snap, node_nz, pod_nz


def test_hand_placements_spread_and_pack(oracle):
    # (1, 0, 1): the first pod scores 87 + 100 on both nodes (node 0 by index); the second 75 + 100 = 175 on node 0
    # against 187 on node 1, and so on alternately.  (0, 1, 0): node 0 always scores higher (25 vs 12, ...).
    snap, node_nz, pod_nz = _two_nodes(4)
    assert pyr.score(1000, 4000, 2 * S.GiB, 8 * S.GiB) == 175 and pyr.score(500, 4000, S.GiB, 8 * S.GiB) == 187
    for w, want in (((1, 0, 1), [0, 1, 0, 1]), ((0, 1, 0), [0, 0, 0, 0])):
        _, node, _, _, nz = rpr.replay_priority(snap, node_nz, pod_nz, None, w)
        assert node.tolist() == want
        assert pyr.replay(snap, None, pyr.PriorityChooser(node_nz, pod_nz, w))[1].tolist() == want
        assert nz[0].tolist() == [500 * want.count(0), 500 * want.count(1)]


def test_hand_placements_busy_node(oracle):
    # node 0 at 2000 m: (1, 0, 1) scores (37 + 87) / 2 + 50 = 112 there against 187 on node 1; (0, 1, 0) scores
    # (62 + 12) / 2 = 37 against 12; first-fit takes node 0
    snap, node_nz, pod_nz = _two_nodes(1, node0_cpu=2000)
    assert pyr.score(2500, 4000, S.GiB, 8 * S.GiB) == 112
    assert pyr.score(2500, 4000, S.GiB, 8 * S.GiB, (0, 1, 0)) == 37
    assert rpr.replay_priority(snap, node_nz, pod_nz, None, (1, 0, 1))[1].tolist() == [1]
    assert rpr.replay_priority(snap, node_nz, pod_nz, None, (0, 1, 0))[1].tolist() == [0]
    assert oracle.replay(snap)[1].tolist() == [0]
