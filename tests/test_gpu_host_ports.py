"""GPU: the PodFitsHostPorts filter (bs_set_host_port_filter) in the round's fit set, bit-exact against the CPU
restatement tests/host_ports_ref.c ANDed with the oracle's fit.  The expectation is the oracle's round on a copy of the
snapshot in which each pod's affinity row is ANDed with the restatement's pass bits (tests/host_ports_ref.py).
Checked: the round's decisions, the fit bitmap, scores, top-K, the priority lists under every default-profile weight
with and without the MatchInterPodAffinity filter, the reason rows and both companions, every lane bound, unaligned
sizes, the designed cases, the switch against no sides at all, the drop rules, every error code, the preemption
refusals, and a random sequence of uploads, row updates and switch flips on one engine.  The walks (bs_replay and
bs_replay_priority, plain and RATIO) are bit-exact per queue position and on the after-state against the hooked walk of
tests/host_ports_ref.c, with fewer and more than 32 representative classes and a negative request; a gang of eight
hostPort workers fits five port-free nodes in the round but not in the walk; LOC runs under the filter."""

import numpy as np
import pytest

import host_port_cases as cases
import host_ports_ref as hr
import interpod_filter_ref as fr
import interpod_priority_ref as ir
import pyref_host_ports as py
import ratio_priority_ref as rr
from randsnap import S, random_snapshot

pytestmark = pytest.mark.gpu

ROUND = ("prefilter", "feasible_count", "best_node", "best_score", "admit", "admit_bitmap", "new_denied", "order", "rank")


def _engine(pkg, snap, cols, on=True, **kw):
    eng = pkg.Engine(snap.lanes, 0, **kw)
    eng.upload(snap)
    if cols is not None:
        eng.upload_host_ports(node=cols[0], pods=cols[1])
    eng.set_host_port_filter(on)
    return eng


def _ok(cols):
    (entries, used), want = cols
    return hr.passes(entries, used, want)


@pytest.mark.parametrize("L", [5, 9, 16])
@pytest.mark.parametrize("P,N", [(200, 500), (77, 1001), (301, 33)])
def test_round_outputs(pkg, oracle, L, P, N):
    snap = random_snapshot(5100 + L + P, P=P, N=N, G=30, L=L, case="mixed")
    cols = hr.random_columns(snap, L + N)
    ok = _ok(cols)
    assert (~ok).any() and ok.any()
    want, fsnap = hr.expected_round(snap, ok, dict(fit_bitmap=True, score=True))
    eng = _engine(pkg, snap, cols, fit_bitmap=True, score=True)
    try:
        res = eng.evaluate()
        for f in ROUND:
            np.testing.assert_array_equal(getattr(res, f), want[f], err_msg=f)
        np.testing.assert_array_equal(eng.fit_rows(), want["fit_rows"])
        np.testing.assert_array_equal(eng.score_rows(), want["score_rows"])
    finally:
        eng.close()


@pytest.mark.parametrize("ipf", [False, True])
@pytest.mark.parametrize("L,P,N", [(5, 200, 500), (9, 77, 1001), (16, 301, 33)])
def test_lists_and_reasons(pkg, oracle, ipf, L, P, N):
    snap = random_snapshot(6100 + L + P, P=P, N=N, G=30, L=L, case="mixed")
    cols = hr.random_columns(snap, 3 * L + N)
    ok = _ok(cols)
    icols = S.node_interpod_filter(snap, L + N, n_zones=6, one_per_host=0.4, ps_affine=0.3, siblings=3) if ipf else None
    iv = fr.verdicts(icols, N) if ipf else None
    want, fsnap = hr.expected_round(snap, ok, dict(reasons=True), ipf_v=iv)
    K = 9
    nz = S.nonzero_requests(snap, 1)
    prefs, loc, spread, ipa = (S.node_preferences(snap, 2), S.node_locality(snap, 3), S.node_spread(snap, 4),
                               S.node_interpod(snap, 5))
    eng = _engine(pkg, snap, cols, fit_bitmap=False, topk=K, reasons=True, priority_k=K)
    eng2 = pkg.Engine(snap.lanes, 0, fit_bitmap=False, topk=K)
    try:
        if ipf:
            eng.upload_interpod_filter(node=icols[0], pods=icols[1])
            eng.set_interpod_filter(True)
        eng.upload_nonzero(node=nz[0], pods=nz[1])
        eng.upload_preferences(node=(prefs[0], prefs[1]), pods=(prefs[2], prefs[3]))
        eng.set_node_priority_weights(1, 1)
        eng.upload_locality(node=loc[0], pods=loc[1])
        eng.set_locality_weights(1, 10000)
        eng.upload_spread(node=spread[0], pods=spread[1])
        eng.set_spread_weight(1)
        eng.upload_interpod(node=ipa[0], pods=ipa[1])
        eng.set_interpod_weight(1)
        res = eng.evaluate()
        for f in ROUND:
            np.testing.assert_array_equal(getattr(res, f), want[f], err_msg=f)
        nodes, scores = eng.priority_rows()
        topk = eng.topk_rows()
        rows, hp_rows = eng.reason_rows(), eng.fetch_host_port_reason_rows()
        ip_rows = eng.fetch_interpod_reason_rows()
        eng2.upload(fsnap)
        eng2.evaluate()
        np.testing.assert_array_equal(topk[0], eng2.topk_rows()[0])
        np.testing.assert_array_equal(topk[1], eng2.topk_rows()[1])
        want_n, want_s = ir.priority_rows(fsnap, nz[0], nz[1], K, ipa, 1, prefs=prefs, pw=(1, 1), loc=loc,
                                          lw=(1, 10000), spread=spread, w_spread=1)
        np.testing.assert_array_equal(nodes, want_n)
        np.testing.assert_array_equal(scores, want_s)
        # the lane rows are the filter-off rows; the companions are the restatements'
        np.testing.assert_array_equal(rows, want["reason_rows"])
        np.testing.assert_array_equal(hp_rows, want["host_port_rows"])
        if ipf:
            np.testing.assert_array_equal(ip_rows, want["interpod_rows"])
        # the ports bin only counts nodes past the guards
        assert (hp_rows + rows[:, 0] + rows[:, 1] <= N).all()
        eng.set_host_port_filter(False)
        eng.evaluate()
        np.testing.assert_array_equal(eng.fetch_host_port_reason_rows(), np.zeros_like(hp_rows))
        np.testing.assert_array_equal(eng.reason_rows(), rows)
    finally:
        eng.close()
        eng2.close()


def test_ports_bin_covers_the_nodes_it_removes(pkg, oracle):
    # every node the filter takes out of a pod's fit set is past the guards and conflicts, so it counts in the ports
    # bin: a node that counts in no bin still fits
    snap = random_snapshot(77, P=120, N=300, G=20, L=5, case="mixed")
    cols = hr.random_columns(snap, 9, grouped=0.6)
    ok = _ok(cols)
    eng = _engine(pkg, snap, cols, fit_bitmap=True, reasons=True)
    try:
        res = eng.evaluate()
        hp_rows = eng.fetch_host_port_reason_rows()
        fit = np.unpackbits(eng.fit_rows().view(np.uint8), axis=1, bitorder="little")[:, :snap.nodes.n].astype(bool)
        plain = oracle.round(snap, want_bitmap=True)
        pfit = np.unpackbits(plain.fit_bitmap.view(np.uint8), axis=1, bitorder="little")[:, :snap.nodes.n].astype(bool)
        np.testing.assert_array_equal(fit, pfit & ok)
        assert ((pfit & ~ok).sum(1) <= hp_rows).all()
        np.testing.assert_array_equal(res.feasible_count, fit.sum(1))
    finally:
        eng.close()


def test_cases_on_device(pkg, oracle):
    # the designed cases: one node per case, every pod fitting it otherwise
    nodes = [py.Node(name, used) for name, used, _, _ in cases.CASES]
    pods = [py.Pod(name, wanted) for name, _, wanted, _ in cases.CASES]
    entries, used, want = py.pack(nodes, pods)
    ok = py.verdicts(pods, nodes)
    np.testing.assert_array_equal(np.diag(ok), [c[3] for c in cases.CASES])
    np.testing.assert_array_equal(hr.passes(entries, used, want), ok)
    base = random_snapshot(9, P=len(pods), N=len(nodes), G=1, L=5, case="mixed")
    eng = _engine(pkg, base, ((entries, used), want), fit_bitmap=True)
    try:
        eng.evaluate()
        on = eng.fit_rows()[:, :1]
        eng.set_host_port_filter(False)
        eng.evaluate()
        off = eng.fit_rows()[:, :1]
    finally:
        eng.close()
    np.testing.assert_array_equal(on, off & fr.pack_bits(ok))


AFTER = ("node_requested", "node_pod_count", "node_req_present", "group_matched", "group_flags", "group_min_res",
         "group_min_res_present", "group_rep_sel", "group_rep_tol")


def _walk_both(pkg, snap, cols, queue=None, nz=None, weights=(1, 0, 1), ratio=None):
    """The engine's walk against host_ports_ref.replay: every queue position and the whole after-state, with the live
    used masks derived from the placements."""
    eng = _engine(pkg, snap, cols)
    try:
        if nz is not None:
            eng.upload_nonzero(node=nz[0], pods=nz[1])
            eng.set_score_weights(*weights)
            if ratio is not None:
                eng.set_ratio_priority(*ratio)
        got = eng.replay(queue, priority=nz is not None)
        got["shape"] = eng.replay_shape()
    finally:
        eng.close()
    pf, node, ready, after, live, nz_live = hr.replay(snap, cols, queue, nz, weights, ratio)
    np.testing.assert_array_equal(got["prefilter"], pf)
    np.testing.assert_array_equal(got["node"], node)
    np.testing.assert_array_equal(got["ready"], ready)
    nt, gt = after.nodes, after.groups
    want = dict(node_requested=nt.requested, node_pod_count=nt.pod_count, node_req_present=nt.req_present,
                group_matched=gt.matched, group_flags=gt.flags, group_min_res=gt.min_res,
                group_min_res_present=gt.min_res_present, group_rep_sel=gt.rep_sel, group_rep_tol=gt.rep_tol)
    for k in AFTER:
        np.testing.assert_array_equal(got[k], want[k], err_msg=k)
    if nz is not None:
        np.testing.assert_array_equal(got["node_nonzero"], nz_live)
    # the live used masks after the walk: the uploaded ones ORed with the want masks of the pods placed on each node
    q = np.arange(snap.pods.n) if queue is None else np.asarray(queue)
    derived = np.array(cols[0][1], np.uint64)
    for qi, n in enumerate(got["node"]):
        if n >= 0:
            derived[n] |= np.uint64(cols[1][q[qi]])
    np.testing.assert_array_equal(derived, live)
    return got


@pytest.mark.parametrize("mode", ["first", "priority", "ratio"])
@pytest.mark.parametrize("L,N,aff", [(5, 300, 0), (9, 1500, 0), (16, 2600, 0), (6, 400, 40)])
def test_walks(pkg, oracle, mode, L, N, aff):
    # aff = 40: more than 32 representative classes (no checkFit bits in the walk)
    snap = random_snapshot(7000 + L + N, P=300, N=N, G=40, L=L, case="mixed", aff=aff)
    cols = hr.random_columns(snap, L * N, grouped=0.5, node_bits=1)
    queue = np.random.default_rng(L).permutation(snap.pods.n) if L % 2 else None
    nz = None if mode == "first" else S.nonzero_requests(snap, L)
    ratio = (2, rr.DEFAULT_SHAPE, [1, 1] + [0] * (L - 2)) if mode == "ratio" else None
    got = _walk_both(pkg, snap, cols, queue, nz, (1, 0, 1), ratio)
    assert (got["node"] >= 0).any()
    assert got["shape"]["fitmask"] == (0 if aff else 1)


def test_walk_negative_request(pkg, oracle):
    # a negative fixed-lane request: the dead-node skip is off (monotone = 0), the port test is unchanged
    snap = random_snapshot(7301, P=200, N=700, G=30, L=5, case="mixed")
    snap.pods.req[0, 3] = -5
    cols = hr.random_columns(snap, 5, grouped=0.5)
    _walk_both(pkg, snap, cols)
    eng = _engine(pkg, snap, cols)
    try:
        eng.replay()
        assert eng.replay_shape()["monotone"] == 0
    finally:
        eng.close()


def _gang(pkg):
    """Eight workers of one gang pin host port 29500 on a cluster of eight roomy nodes, three of which hold it."""
    snap = random_snapshot(31, P=8, N=8, G=1, L=5, case="mixed")
    nt, pt, gt = snap.nodes, snap.pods, snap.groups
    nt.flags[:] = 0
    nt.label_mask[:] = 0
    nt.taint_mask[:] = 0
    nt.alloc[:4] = 1 << 40
    nt.requested[:] = 0
    nt.pod_count[:] = 0
    nt.alloc_present[:] = 0xF
    nt.req_present[:] = 0
    pt.req[:] = 1
    pt.req_present[:] = 0xF
    pt.gid[:] = 0
    pt.flags[:] = 0
    pt.sel_mask[:] = 0
    pt.tol_mask[:] = 0
    if pt.aff_class is not None:
        pt.aff_class[:] = 0xFFFFFFFF
    gt.min_member[:] = 8
    gt.scheduled[:] = 0
    gt.matched[:] = 0
    gt.flags[:] = 0
    nodes = [py.Node(f"n{i}", [py.Port(29500)] if i >= 5 else []) for i in range(8)]
    pods = [py.Pod(f"w{i}", [py.Port(29500)]) for i in range(8)]
    entries, used, want = py.pack(nodes, pods)
    return snap, ((entries, used), want)


def test_hostport_gang(pkg, oracle):
    # the round admits the gang (each worker alone fits a port-free node); the walk places one worker per port-free
    # node, five in all, and the gang stays waiting, as upstream would leave it
    snap, cols = _gang(pkg)
    ok = _ok(cols)
    assert ok[:, :5].all() and not ok[:, 5:].any()
    want_round, _ = hr.expected_round(snap, ok, dict(fit_bitmap=True))
    eng = _engine(pkg, snap, cols, fit_bitmap=True)
    try:
        res = eng.evaluate()
        for f in ROUND:
            np.testing.assert_array_equal(getattr(res, f), want_round[f], err_msg=f)
        assert (res.feasible_count == 5).all() and res.admit[0] == fr.ADMIT
    finally:
        eng.close()
    got = _walk_both(pkg, snap, cols)
    assert sorted(got["node"][got["node"] >= 0].tolist()) == [0, 1, 2, 3, 4]
    assert not got["ready"].any()
    # without the filter the walk stacks all eight on the roomy nodes and the gang is ready
    eng = _engine(pkg, snap, cols, on=False)
    try:
        off = eng.replay()
    finally:
        eng.close()
    assert (off["node"] >= 0).all() and off["ready"][-1] == 1


def test_walk_with_locality(pkg, oracle):
    # LOC under the filter: every placement avoids a conflict, and with no wanted ports the walk is the filter-off one
    snap = random_snapshot(7401, P=200, N=600, G=30, L=5, case="mixed")
    cols = hr.random_columns(snap, 8, grouped=0.6, node_bits=1)
    nz, loc = S.nonzero_requests(snap, 2), S.node_locality(snap, 3)
    outs = []
    for c in (cols, (cols[0], np.zeros_like(cols[1])), None):
        eng = _engine(pkg, snap, c, on=c is not None)
        try:
            eng.upload_nonzero(node=nz[0], pods=nz[1])
            eng.upload_locality(node=loc[0], pods=loc[1])
            eng.set_locality_weights(1, 10000)
            outs.append(eng.replay(priority=True))
        finally:
            eng.close()
    (entries, used), want = cols
    live = np.array(used, np.uint64)
    for p, n in enumerate(outs[0]["node"]):
        if n >= 0:
            assert hr.passes(entries, live[n:n + 1], want[p:p + 1])[0, 0]
            live[n] |= np.uint64(want[p])
    for k in ("prefilter", "node", "ready"):
        np.testing.assert_array_equal(outs[1][k], outs[2][k])


def test_switch_off_is_no_sides(pkg, oracle):
    snap = random_snapshot(525, P=150, N=300, G=20, L=9, case="mixed")
    cols = hr.random_columns(snap, 3)
    outs = []
    for sides in (False, True):
        eng = _engine(pkg, snap, cols if sides else None, on=False, fit_bitmap=True, score=True, reasons=True)
        try:
            res = eng.evaluate()
            outs.append([getattr(res, f).copy() for f in ROUND] + [eng.fit_rows(), eng.score_rows(), eng.reason_rows()])
            if sides:   # on, then off again: the filter-off outputs once more
                eng.set_host_port_filter(True)
                eng.evaluate()
                eng.set_host_port_filter(False)
                res = eng.evaluate()
                outs.append([getattr(res, f).copy() for f in ROUND] + [eng.fit_rows(), eng.score_rows(),
                                                                       eng.reason_rows()])
        finally:
            eng.close()
    for a, b in zip(outs[0], outs[1]):
        np.testing.assert_array_equal(a, b)
    for a, b in zip(outs[0], outs[2]):
        np.testing.assert_array_equal(a, b)


def _code(pkg, fn, *a):
    with pytest.raises(pkg.capi.BsError) as ei:
        fn(*a)
    return ei.value.code


def test_drop_rules_and_errors(pkg, oracle):
    capi = pkg.capi
    snap = random_snapshot(727, P=60, N=100, G=10, L=5, case="mixed")
    cols = hr.random_columns(snap, 6)
    (entries, used), want = cols
    eng = _engine(pkg, snap, cols)
    try:
        eng.evaluate()
        eng.upload_nodes(snap.nodes)   # drops the node side
        assert _code(pkg, eng.evaluate) == capi.BS_E_STATE
        eng.upload_host_ports(node=cols[0])
        eng.evaluate()
        eng.update_nodes(np.array([0], np.uint32), snap.nodes.take(np.array([0])))   # drops it too
        assert _code(pkg, eng.evaluate) == capi.BS_E_STATE
        eng.upload_host_ports(node=cols[0])
        eng.upload_pods(snap.pods)     # drops the pod side
        assert _code(pkg, eng.evaluate) == capi.BS_E_STATE
        eng.upload_host_ports(pods=want)
        eng.evaluate()
        K = len(entries)
        bad_node = [
            ((entries, used[:-1]), capi.BS_E_INVAL),                                          # n_nodes
            ((np.concatenate([entries, entries[:1]]), used), capi.BS_E_INVAL),                # a duplicate
            ((np.array([[k, 0, 1000 + k] for k in range(65)]), np.zeros_like(used)), capi.BS_E_INVAL),   # 65 entries
            ((np.concatenate([entries[:-1], [[0, 0, 0]]]), used), capi.BS_E_RANGE),           # port 0
            ((np.concatenate([entries[:-1], [[0, 0, 65536]]]), used), capi.BS_E_RANGE),       # port 65536
            ((entries, used | np.uint64(1 << K)), capi.BS_E_INDEX),                           # a used bit >= K
        ]
        for b, code in bad_node:
            assert _code(pkg, eng.upload_host_ports, b, None) == code
            assert _code(pkg, eng.evaluate) == capi.BS_E_STATE   # a failing upload leaves the side dropped
        # exactly 64 entries is accepted
        eng.upload_host_ports(node=(np.array([[k, 0, 1000 + k] for k in range(64)]), np.zeros_like(used)))
        eng.upload_host_ports(node=cols[0])
        assert _code(pkg, eng.upload_host_ports, None, want[:-1]) == capi.BS_E_INVAL
        assert _code(pkg, eng.evaluate) == capi.BS_E_STATE
        # a want bit outside the dictionary: refused at evaluation, in either upload order
        eng.upload_host_ports(pods=want | np.uint64(1 << K))
        assert _code(pkg, eng.evaluate) == capi.BS_E_INDEX
        eng.upload_host_ports(node=(np.concatenate([entries, [[7, 1, 4242]]]), used))
        eng.evaluate()
        eng.upload_host_ports(node=cols[0], pods=want)
        eng.evaluate()
        # no side at all, switch on: BS_E_STATE
        eng2 = _engine(pkg, snap, None)
        try:
            assert _code(pkg, eng2.evaluate) == capi.BS_E_STATE
            assert "PodFitsHostPorts" in eng2.lib.bs_last_error(eng2.h).decode()
        finally:
            eng2.close()
    finally:
        eng.close()


def test_refusals(pkg, oracle):
    snap = random_snapshot(828, P=40, N=60, G=8, L=5, case="mixed")
    cols = hr.random_columns(snap, 7)
    eng = _engine(pkg, snap, cols)
    try:
        eng.evaluate()
        calls = [lambda: eng.preempt(np.array([0], np.uint32)), lambda: eng.preempt_walk(np.array([0], np.uint32))]
        assert [_code(pkg, c) for c in calls] == [pkg.capi.BS_E_INVAL] * 2
        assert "PodFitsHostPorts" in eng.lib.bs_last_error(eng.h).decode()
        # the walks check the sides as a round does, before anything launches
        eng.upload_nodes(snap.nodes)
        assert _code(pkg, eng.replay) == pkg.capi.BS_E_STATE
        eng.upload_host_ports(node=cols[0], pods=cols[1] | np.uint64(1 << 40))
        assert _code(pkg, eng.replay) == pkg.capi.BS_E_INDEX
    finally:
        eng.close()


def test_random_sequence(pkg, oracle):
    # uploads, row updates, pod-side re-uploads and switch flips on one long-lived engine; every round's fit rows are
    # the filter-off rows ANDed with the restatement while the filter is on
    snap = random_snapshot(939, P=250, N=180, G=30, L=5, case="mixed")
    rng = np.random.default_rng(4)
    W = (snap.nodes.n + 31) // 32
    eng = pkg.Engine(snap.lanes, 0, fit_bitmap=True)
    ref = pkg.Engine(snap.lanes, 0, fit_bitmap=True)
    try:
        eng.upload(snap)
        ref.upload(snap)
        cols = hr.random_columns(snap, 100)
        eng.upload_host_ports(node=cols[0], pods=cols[1])
        on = False
        for k in range(30):
            op = rng.integers(0, 4)
            if op == 0:
                on = not on
                eng.set_host_port_filter(on)
            elif op == 1:
                cols = (cols[0], hr.random_columns(snap, 200 + k, grouped=float(rng.random()))[1])
                eng.upload_host_ports(pods=cols[1])
            elif op == 2:
                cols = (hr.random_columns(snap, 300 + k)[0], cols[1])
                eng.upload_host_ports(node=cols[0], pods=cols[1])
            else:
                idx = np.sort(rng.choice(snap.nodes.n, 5, replace=False)).astype(np.uint32)
                rows = snap.nodes.take(idx)
                eng.update_nodes(idx, rows)
                ref.update_nodes(idx, rows)
                if on:
                    assert _code(pkg, eng.evaluate) == pkg.capi.BS_E_STATE
                eng.upload_host_ports(node=cols[0])
            eng.evaluate()
            ref.evaluate()
            got, off = eng.fit_rows()[:, :W], ref.fit_rows()[:, :W]
            np.testing.assert_array_equal(got, off & fr.pack_bits(_ok(cols)) if on else off, err_msg=str(k))
    finally:
        eng.close()
        ref.close()
