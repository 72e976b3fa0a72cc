"""GPU: the MatchInterPodAffinity filter in the walks (bs_replay, bs_replay_priority) on live presence, bit-exact per
queue position and on the whole after-state against tests/interpod_walk_ref.c's hook pair around the oracle's walk:
first fit, priority, RATIO and LOC, with PodFitsHostPorts off and on, every MAXL build, on snapshot.node_interpod_walk's
columns.  Also: the first step's fit set is the round's fit row, a round after a walk is unchanged, the hand-built cases and a
parameter server with hostPort workers, and every refusal of the placed side."""

import numpy as np
import pytest

import host_ports_ref as hr
import interpod_filter_ref as fr
import interpod_walk_cases as cases
import interpod_walk_ref as iwr
import pyref_interpod_filter as pyf
import pyref_interpod_walk as pyw
import ratio_priority_ref as rr
from randsnap import S, random_snapshot

pytestmark = pytest.mark.gpu

ROUND = ("prefilter", "feasible_count", "best_node", "best_score", "admit", "admit_bitmap", "new_denied", "order", "rank")
AFTER = ("node_requested", "node_pod_count", "node_req_present", "group_matched", "group_flags", "group_min_res",
         "group_min_res_present", "group_rep_sel", "group_rep_tol")


def _engine(pkg, snap, cols, placed, hp=None, **kw):
    eng = pkg.Engine(snap.lanes, 0, **kw)
    eng.upload(snap)
    eng.upload_interpod_filter(node=cols[0], pods=cols[1])
    eng.set_interpod_filter(True)
    if placed is not None:
        eng.upload_interpod_placed(*placed)
    if hp is not None:
        eng.upload_host_ports(node=hp[0], pods=hp[1])
        eng.set_host_port_filter(True)
    return eng


def _code(pkg, fn, *a):
    with pytest.raises(pkg.capi.BsError) as ei:
        fn(*a)
    return ei.value.code


def _walk_both(pkg, snap, cols, placed, queue=None, mode="first", hp=None, L=5):
    """The engine's walk against interpod_walk_ref.replay: every queue position and the whole after-state."""
    nz = None if mode == "first" else S.nonzero_requests(snap, L)
    ratio = (2, rr.DEFAULT_SHAPE, [1, 1] + [0] * (snap.lanes - 2)) if mode == "ratio" else None
    loc = S.node_locality(snap, 3) if mode == "loc" else None
    lw = (1, 10000) if mode == "loc" else (0, 0)
    eng = _engine(pkg, snap, cols, placed, hp, fit_bitmap=True)
    try:
        if nz is not None:
            eng.upload_nonzero(node=nz[0], pods=nz[1])
            eng.set_score_weights(1, 0, 1)
        if ratio is not None:
            eng.set_ratio_priority(*ratio)
        if loc is not None:
            eng.upload_locality(node=loc[0], pods=loc[1])
            eng.set_locality_weights(*lw)
        before = eng.evaluate()
        before = {f: getattr(before, f).copy() for f in ROUND}
        fit_before = eng.fit_rows().copy()
        got = eng.replay(queue, priority=nz is not None)
        after = eng.evaluate()
        # the walk leaves the uploaded sides as they were: the round after it is the round before it
        for f in ROUND:
            np.testing.assert_array_equal(getattr(after, f), before[f], err_msg=f)
        np.testing.assert_array_equal(eng.fit_rows(), fit_before)
    finally:
        eng.close()
    pf, node, ready, snap_after, nz_live, hp_live = iwr.replay(snap, cols, placed, queue, nz, (1, 0, 1), ratio, loc,
                                                               lw, hp)
    np.testing.assert_array_equal(got["prefilter"], pf)
    np.testing.assert_array_equal(got["node"], node)
    np.testing.assert_array_equal(got["ready"], ready)
    nt, gt = snap_after.nodes, snap_after.groups
    want = dict(node_requested=nt.requested, node_pod_count=nt.pod_count, node_req_present=nt.req_present,
                group_matched=gt.matched, group_flags=gt.flags, group_min_res=gt.min_res,
                group_min_res_present=gt.min_res_present, group_rep_sel=gt.rep_sel, group_rep_tol=gt.rep_tol)
    for k in AFTER:
        np.testing.assert_array_equal(got[k], want[k], err_msg=k)
    if nz is not None:
        np.testing.assert_array_equal(got["node_nonzero"], nz_live)
    # the first step sees the round's verdicts: a passing pod goes to a node of its round fit row (first fit: the first
    # one), and to none when the row is empty; test_first_step_fit_set compares whole sets
    q0 = 0 if queue is None else int(queue[0])
    if got["prefilter"][0] == 0:
        fits = np.flatnonzero(np.unpackbits(fit_before[q0].view(np.uint8), bitorder="little")[:snap.nodes.n])
        if mode == "first":
            assert got["node"][0] == (fits[0] if len(fits) else -1)
        else:
            assert got["node"][0] in fits if len(fits) else got["node"][0] == -1
    return got


def test_first_step_fit_set(pkg, oracle):
    # the whole fit set of a walk's first step equals the round's fit row: first fit over the nodes from k on (those
    # before k flagged unschedulable) returns the next node of the set after k - 1, so the set is enumerated node by
    # node.  The pods are taken out of their gangs so that PreFilter passes whatever the flags.
    snap = random_snapshot(8400, P=80, N=150, G=12, L=5, case="mixed")
    node, pods, placed = S.node_interpod_walk(snap, 11, n_zones=4, one_per_host=0.5, ps_affine=0.3, siblings=3)
    picks = [int(p) for p in np.flatnonzero(pods[0] != pyf.IPF_NONE)[:4]]
    assert picks
    snap.pods.gid[picks] = S.GID_NONE
    eng = _engine(pkg, snap, (node, pods), placed, fit_bitmap=True)
    try:
        eng.evaluate()
        rows = eng.fit_rows().copy()
        for p in picks:
            want = np.flatnonzero(np.unpackbits(rows[p].view(np.uint8), bitorder="little")[:snap.nodes.n]).tolist()
            got, k = [], 0
            while k < snap.nodes.n:
                s2 = snap.copy()
                s2.nodes.flags[:k] |= S.NODE_UNSCHEDULABLE
                eng.upload(s2)
                eng.upload_interpod_filter(node=node, pods=pods)
                eng.upload_interpod_placed(*placed)
                n = int(eng.replay(np.array([p], np.uint32), after_state=False)["node"][0])
                if n < 0:
                    break
                got.append(n)
                k = n + 1
            assert got == want, p
        assert any(len(np.flatnonzero(rows[p])) for p in picks)
    finally:
        eng.close()


@pytest.mark.parametrize("hp", [False, True])
@pytest.mark.parametrize("mode", ["first", "priority", "ratio", "loc"])
@pytest.mark.parametrize("L,N", [(5, 300), (9, 500), (16, 400)])
def test_walks(pkg, oracle, L, N, mode, hp):
    snap = random_snapshot(8100 + L + N, P=200, N=N, G=30, L=L, case="mixed")
    node, pods, placed = S.node_interpod_walk(snap, L + N, n_zones=4, one_per_host=0.4, ps_affine=0.3, siblings=2,
                                              filler=1, n_blockers=8)
    hcols = hr.random_columns(snap, L * N, grouped=0.4, node_bits=1) if hp else None
    queue = np.random.default_rng(L + N).permutation(snap.pods.n).astype(np.uint32) if L != 9 else None
    got = _walk_both(pkg, snap, (node, pods), placed, queue, mode, hcols, L)
    assert (got["node"] >= 0).any()


def test_filter_changes_placements(pkg, oracle):
    # the seeded columns keep some pods out that the walk without the filter places
    snap = random_snapshot(8200, P=200, N=300, G=30, L=5, case="mixed")
    node, pods, placed = S.node_interpod_walk(snap, 3, n_zones=4, one_per_host=0.6, ps_affine=0.3, siblings=2, filler=1)
    on = _walk_both(pkg, snap, (node, pods), placed)
    eng = pkg.Engine(snap.lanes, 0)
    try:
        eng.upload(snap)
        off = eng.replay()
    finally:
        eng.close()
    assert ((on["node"] < 0) & (off["node"] >= 0)).any()


@pytest.mark.parametrize("case", cases.CASES, ids=[c[0] for c in cases.CASES])
def test_cases_on_device(pkg, oracle, case):
    name, nodes, existing, pending, _, want = case
    snap = cases.snapshot(len(nodes), len(pending))
    cols = pyf.pack(nodes, existing, pending)
    placed = pyw.placed(nodes, existing, pending)
    queue = cases.queue_of(case)
    got = _walk_both(pkg, snap, cols, placed, queue)
    assert got["node"].tolist() == want
    if name == "eight-anti-workers":
        # each worker alone fits five hosts: the round admits the gang, the walk leaves it waiting
        eng = _engine(pkg, snap, cols, placed)
        try:
            res = eng.evaluate()
        finally:
            eng.close()
        assert (res.feasible_count == 5).all() and res.admit[0] == fr.ADMIT
        assert not got["ready"].any()


def test_ps_and_hostport_workers(pkg, oracle):
    # the parameter server first, then three hostPort workers that need its zone: one worker per port-free host of
    # zone b, with both filters on
    nodes = cases._nodes("b", "a", "b", "b")
    pending = [cases._ps()] + [cases._follower(f"w{i}") for i in range(3)]
    snap = cases.snapshot(len(nodes), len(pending))
    cols = pyf.pack(nodes, [], pending)
    placed = pyw.placed(nodes, [], pending)
    hp = ((np.array([[0, 0, 29500]], np.int64), np.zeros(len(nodes), np.uint64)),
          np.array([0, 1, 1, 1], np.uint64))
    got = _walk_both(pkg, snap, cols, placed, hp=hp)
    assert got["node"].tolist() == [0, 0, 2, 3]
    assert got["ready"][-1] == 1


def test_refusals(pkg, oracle):
    capi = pkg.capi
    snap = random_snapshot(8300, P=60, N=100, G=10, L=5, case="mixed")
    node, pods, placed = S.node_interpod_walk(snap, 5)
    P, T = snap.pods.n, len(node[2])
    pcls, (qoff, qterm, qown, qmatch) = placed
    assert len(qterm)
    eng = _engine(pkg, snap, (node, pods), None)
    try:
        eng.upload_nonzero(*S.nonzero_requests(snap, 1))
        walks = [lambda: eng.replay(), lambda: eng.replay(priority=True)]
        # no placed side: both walks refuse as before, and name the call that uploads it
        for w in walks:
            assert _code(pkg, w) == capi.BS_E_INVAL
            msg = eng.lib.bs_last_error(eng.h).decode()
            assert "MatchInterPodAffinity" in msg and "bs_upload_pod_interpod_placed" in msg
        eng.upload_interpod_placed(*placed)
        ok = eng.replay()
        # uploading pods drops the side
        eng.upload(snap)
        eng.upload_interpod_filter(node=node, pods=pods)
        eng.upload_nonzero(*S.nonzero_requests(snap, 1))
        assert _code(pkg, eng.replay) == capi.BS_E_INVAL
        eng.upload_interpod_placed(*placed)
        np.testing.assert_array_equal(eng.replay()["node"], ok["node"])
        # a term outside the dictionary: accepted here, refused when a walk starts
        eng.upload_interpod_placed(pcls, (qoff, np.where(np.arange(len(qterm)) == 0, T, qterm), qown, qmatch))
        for w in walks:
            assert _code(pkg, w) == capi.BS_E_INDEX
        bad = [
            (capi.BS_E_INVAL, (pcls[:-1], (qoff, qterm, qown, qmatch))),                       # n_pods
            (capi.BS_E_INVAL, (pcls, (qoff[::-1].copy(), qterm, qown, qmatch))),              # offsets
            (capi.BS_E_INDEX, (np.full(P, len(qoff) - 1, np.uint32), (qoff, qterm, qown, qmatch))),   # pod_class
            (capi.BS_E_RANGE, (pcls, (qoff, qterm, np.full_like(qown, 2), qmatch))),          # own 2
            (capi.BS_E_RANGE, (pcls, (qoff, qterm, qown, np.full_like(qmatch, 2)))),          # match 2
        ]
        for code, args in bad:
            eng.upload_interpod_placed(*placed)
            assert _code(pkg, eng.upload_interpod_placed, *args) == code
            assert _code(pkg, eng.replay) == capi.BS_E_INVAL   # a failing call leaves the side dropped
        # preemption still refuses under the filter
        assert _code(pkg, eng.preempt, np.array([0], np.uint32)) == capi.BS_E_INVAL
        # with the filter off the placed side changes nothing
        eng.set_interpod_filter(False)
        off_without = eng.replay()
        eng.upload_interpod_placed(*placed)
        off_with = eng.replay()
        for k in ("prefilter", "node", "ready") + AFTER:
            np.testing.assert_array_equal(off_with[k], off_without[k], err_msg=k)
    finally:
        eng.close()
