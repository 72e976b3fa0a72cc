"""CPU: every designed case of tests/replay_regime_cases.py holds the property it was built for, checked with the
oracle and with replay_walk's host rule restated: the regime each case claims, the block where the cache-limit
cases first meet their need, the border case's verdict flip, the dead-node survivor and where it is placed, the
findMaxPG buckets and where their ties sit, and the panic position.  A case that loses its property fails here."""
import numpy as np
import pytest

import replay_regime_cases as rc
from randsnap import S

CASES = rc.cases()


@pytest.mark.parametrize("name", list(CASES))
def test_claimed_regime_is_the_host_rule(name):
    c = CASES[name]
    got = rc.regime(c.snap, len(c.queue))
    for k, v in c.regime.items():
        if k != "lo":
            assert got[k] == v, k


def _first_met(nt, need, percent):
    """Index of the first node prefix whose fixed-lane residuals meet `need` (every node is visible and fits)."""
    from oracle import oracle
    run = np.ones(nt.n, bool)
    for d in range(4):
        caps = np.unique(nt.alloc[d])
        scaled = dict(zip(caps.tolist(), (oracle.scale(int(v), percent) for v in caps)))
        sub = nt.pod_count.astype(np.int64) if d == S.LANE_PODS else nt.requested[d]
        left = np.vectorize(scaled.get, otypes=[np.int64])(nt.alloc[d]) - sub
        run &= np.cumsum(left) >= need[d]
    return int(np.argmax(run)) if run.any() else None


@pytest.mark.parametrize("name", [n for n in CASES if n.startswith("cache_")])
def test_cache_limit_need_met_in_the_last_block(name, oracle):
    c = CASES[name]
    nt, gt, pt = c.snap.nodes, c.snap.groups, c.snap.pods
    assert not nt.flags.any() and (nt.label_mask == 0xF).all() and not nt.taint_mask.any()
    # the first check: pod 0's own group (case A) or the max group plus the pod (case B)
    p = int(c.queue[np.flatnonzero(pt.gid[c.queue] >= 0)[0]])
    g = int(pt.gid[p])
    m, _, _ = oracle.find_max_pg(gt)
    need = np.zeros(4, np.int64)
    if gt.matched[m] == 0:
        assert c.info["percent"] == 1.0
        need[:3] = gt.min_res[:3, g] * (int(gt.min_member[g]) - int(gt.scheduled[g]))
        need[3] = gt.min_member[g] + 1 if need[3] == 0 else need[3]
    else:
        assert c.info["percent"] == 0.7
        nf = int(gt.min_member[m]) - int(gt.matched[m])
        need[:4] = gt.min_res[:4, m] * max(nf, 0) + pt.req[:4, p]
        if gt.min_res[3, m] * max(nf, 0) == 0:
            need[3] = gt.min_member[m] + 1 + pt.req[3, p]
    at = _first_met(nt, need, c.info["percent"])
    assert at is not None and at // rc.BLOCK == 1023 and at >= c.info["head"]
    # pods are assumed into that block partway through the walk, and checks follow them
    pf, node, _, _ = oracle.replay(c.snap, c.queue)
    placed = np.flatnonzero(node >= 0)
    assert len(placed) >= 2 and (node[placed] >= c.info["head"]).all() and (node[placed] // rc.BLOCK == 1023).all()
    assert (pf[placed[0] + 1:] != S.PF_PASS).any() or (pt.gid[c.queue[placed[0] + 1:]] >= 0).any()


@pytest.mark.parametrize("n", [31, 32, 33])
def test_class_border_flips_the_verdict(n, oracle):
    c = CASES[f"classes_{n}"]
    snap = c.snap
    assert rc.rep_classes(snap) == n
    # group 0's class is the last id: pods' classes first, then the groups' new ones
    pod_keys = set(zip(snap.pods.sel_mask.tolist(), snap.pods.tol_mask.tolist()))
    assert (int(snap.groups.rep_sel[0]), int(snap.groups.rep_tol[0])) not in pod_keys and len(pod_keys) == n - 1
    total = c.info["total"]
    need = np.array([total, 0, 0, 2, 0], np.int64)
    assert oracle.compare_cluster(snap.nodes, 0, 1000, need, 0, 1.0)
    short = snap.nodes.copy()
    short.requested[0, 1] += 1
    assert not oracle.compare_cluster(short, 0, 1000, need, 0, 1.0)   # one unit fewer anywhere: not enough
    assert _first_met(snap.nodes, need[:4], 1.0) == rc.BORDER_N - 1    # met only by the last node of block 1
    pf, node, _, _ = oracle.replay(snap, c.queue)
    assert pf.tolist() == [S.PF_PASS, S.PF_PASS, S.PF_NOT_ENOUGH] and node.tolist() == [-1, 1, -1]


@pytest.mark.parametrize("variant", ["edge", "below", "negative"])
def test_dead_node_survivor(variant, oracle):
    c = CASES[f"dead_{variant}"]
    nt, pt = c.snap.nodes, c.snap.pods
    min_cpu = int(pt.req[0].min())
    pos_min = int(pt.req[0][pt.req[0] > 0].min())
    assert pos_min == rc.SMALL_CPU and (min_cpu < 0) == (variant == "negative")
    left = nt.alloc[0, :rc.BLOCK] - nt.requested[0, :rc.BLOCK]
    others = np.delete(left, rc.SURVIVOR)
    assert (others < pos_min).all()
    assert left[rc.SURVIVOR] == pos_min - (variant == "below")
    # nothing else makes a block-0 node dead: every other fixed lane has room for any pod of the table
    for d in (1, 2):
        assert ((nt.alloc[d] - nt.requested[d]) >= pt.req[d].max()).all()
    assert ((nt.alloc[3] - nt.pod_count) >= 1).all() and not pt.req[3].any()
    # early pods ask for more than the survivor leaves; the smallest comes last
    assert (pt.req[0, c.queue[:-1]] > pos_min).all() and pt.req[0, c.queue[-1]] == pos_min
    pf, node, _, _ = oracle.replay(c.snap, c.queue)
    assert (pf == S.PF_PASS).all() and (node[:-1] >= rc.BLOCK).all()
    if variant == "below":
        assert node[-1] >= rc.BLOCK
    else:
        assert node[-1] == rc.SURVIVOR


def _finished(gt, g):
    mm, sc = int(gt.min_member[g]), int(gt.scheduled[g])
    if (mm - sc) % 2**32 == 0:
        return 0
    return ((int(gt.matched[g]) + sc) % 2**32 * 1000) % 2**32 // mm


@pytest.mark.parametrize("G", [32768, 32769, 100000])
@pytest.mark.parametrize("case", ["A", "B"])
def test_bucket_borders_and_ties(G, case, oracle):
    c = CASES[f"buckets_{case}_G{G}"]
    gt = c.snap.groups
    size, nb = rc.buckets(G)
    assert (size, nb) == {32768: (32, 1024), 32769: (64, 513), 100000: (128, 782)}[G]
    assert G - (nb - 1) * size == {32768: 32, 32769: 1, 100000: 32}[G]     # groups in the last bucket
    t0, t1, t3 = c.info["keys"]
    assert t0 // size < t1 // size < t3 // size == nb - 1
    if size > 32:
        assert t0 % size >= 32 and t1 % size >= 32   # past the first 32 groups of their bucket
    tie = c.info["tie"]
    assert [_finished(gt, g) for g in (t0, t1, t3)] == [tie] * 3
    # t0 may be replaced (scheduled >= min_member), t1 then keeps the maximum against t3 (scheduled 0)
    assert gt.scheduled[t0] >= gt.min_member[t0] and gt.scheduled[t1] == 0 and gt.scheduled[t3] == 0
    visible = (gt.flags & S.GROUP_HAS_POD).astype(bool) & ~(gt.flags & S.GROUP_SCHEDULED).astype(bool)
    assert np.flatnonzero(visible).tolist() == [t0, t1, t3]
    assert oracle.find_max_pg(gt)[:2] == (t1, tie)
    # every other group stays below the tie when its first pod arrives
    others = np.setdiff1d(np.arange(G), [t0, t1, t3])
    fin = (gt.matched[others].astype(np.int64) * 1000) // gt.min_member[others]
    assert (fin < max(tie, 1000)).all()
    if case == "B":
        assert not (c.snap.nodes.label_mask & np.uint64(rc.UNFIT_SEL)).any() and gt.rep_sel[t1] == rc.UNFIT_SEL
        pf, node, _, _ = oracle.replay(c.snap, c.queue)
        assert (pf == S.PF_NOT_ENOUGH).any() and (node >= 0).any()


@pytest.mark.parametrize("variant", ["panic", "quiet", "zero"])
def test_panic_position(variant, oracle):
    c = CASES[f"panic_{variant}"]
    pt, gt = c.snap.pods, c.snap.groups
    at = list(c.queue).index(10)
    assert pt.gid[10] == 2 and pt.flags[10] & S.POD_OCC_NOREFS and gt.min_member[2] == 0
    assert not gt.flags[2] & S.GROUP_HAS_POD and list(c.queue).count(10) == 1
    pf, node, ready, _, panic = oracle.replay(c.snap, c.queue, panic=True)
    assert pf[at] == S.PF_OCC_NOREFS
    assert panic == c.panic_at
    if variant == "panic":
        assert panic == at + 1
    # the four-value form is unchanged
    pf4, node4, ready4, _ = oracle.replay(c.snap, c.queue)
    assert (pf4 == pf).all() and (node4 == node).all() and (ready4 == ready).all()
