"""GPU: the MatchInterPodAffinity filter (bs_set_interpod_filter) in the round's fit set, bit-exact against the CPU
restatement tests/interpod_filter_ref.c ANDed with the oracle's fit.  The expectation is the oracle's round on a copy of
the snapshot in which each pod gets an affinity row of its own, its old row ANDed with the restatement's pass bits: the
filter is a per-pod node predicate that PreFilter never reads, so every fit-set output of that round is the filter's.
Checked: the round's decisions, the fit bitmap, scores, top-K, the priority lists under every default-profile weight,
the reason rows and their companion, every lane bound, unaligned sizes, more than 32768 filter classes, the switch
against no sides at all, when the pre-pass runs, the drop rules, the caps and error codes, the four refusals, and
sampled pods of a cfg4 round with the generator's columns."""

import numpy as np
import pytest

import interpod_filter_cases as cases
import interpod_filter_ref as fr
import interpod_priority_ref as ir
import pyref_interpod_filter as py
from randsnap import S, random_snapshot

pytestmark = pytest.mark.gpu

def _engine(pkg, snap, cols, on=True, **kw):
    eng = pkg.Engine(snap.lanes, 0, **kw)
    eng.upload(snap)
    if cols is not None:
        eng.upload_interpod_filter(node=cols[0], pods=cols[1])
    eng.set_interpod_filter(on)
    return eng


ROUND = ("prefilter", "feasible_count", "best_node", "best_score", "admit", "admit_bitmap", "new_denied", "order", "rank")


def _check_round(pkg, oracle, snap, cols):
    """The round under the filter against interpod_filter_ref.expected_round: the fit-set outputs are the filtered
    snapshot's, PreFilter's (and the sort's) the plain snapshot's (a pod's affinity row also reaches PreFilter, the
    filter does not), and Permit readiness follows from both."""
    want, fsnap = fr.expected_round(snap, cols, dict(fit_bitmap=True, score=True))
    eng = _engine(pkg, snap, cols, fit_bitmap=True, score=True)
    try:
        res = eng.evaluate()
        for f in ROUND:
            np.testing.assert_array_equal(getattr(res, f), want[f], err_msg=f)
        np.testing.assert_array_equal(eng.fit_rows(), want["fit_rows"])
        np.testing.assert_array_equal(eng.score_rows(), want["score_rows"])
    finally:
        eng.close()
    return fr.verdicts(cols, snap.nodes.n), fsnap, oracle.round(snap, want_bitmap=True)


@pytest.mark.parametrize("L", [5, 9, 16])
@pytest.mark.parametrize("P,N", [(200, 500), (77, 1001), (301, 33)])
def test_round_outputs(pkg, oracle, L, P, N):
    snap = random_snapshot(4100 + L + P, P=P, N=N, G=30, L=L, case="mixed")
    cols = S.node_interpod_filter(snap, L + N, n_zones=6, one_per_host=0.4, ps_affine=0.3, siblings=3)
    v, fsnap, plain = _check_round(pkg, oracle, snap, cols)
    assert (v != fr.PASS).any()
    # top-K, reason rows and companion rows, priority lists with every default-profile weight on
    K = 9
    nz = S.nonzero_requests(snap, 1)
    prefs, loc, spread, ipa = (S.node_preferences(snap, 2), S.node_locality(snap, 3), S.node_spread(snap, 4),
                               S.node_interpod(snap, 5))
    eng = _engine(pkg, snap, cols, fit_bitmap=False, topk=K, reasons=True, priority_k=K)
    eng2 = pkg.Engine(snap.lanes, 0, fit_bitmap=False, topk=K)
    try:
        eng.upload_nonzero(node=nz[0], pods=nz[1])
        eng.upload_preferences(node=(prefs[0], prefs[1]), pods=(prefs[2], prefs[3]))
        eng.set_node_priority_weights(1, 1)
        eng.upload_locality(node=loc[0], pods=loc[1])
        eng.set_locality_weights(1, 10000)
        eng.upload_spread(node=spread[0], pods=spread[1])
        eng.set_spread_weight(1)
        eng.upload_interpod(node=ipa[0], pods=ipa[1])
        eng.set_interpod_weight(1)
        eng.evaluate()
        nodes, scores = eng.priority_rows()
        topk = eng.topk_rows()
        rows, comp = eng.reason_rows(), eng.fetch_interpod_reason_rows()
        eng2.upload(fsnap)
        eng2.evaluate()
        np.testing.assert_array_equal(topk[0], eng2.topk_rows()[0])
        np.testing.assert_array_equal(topk[1], eng2.topk_rows()[1])
        want_n, want_s = ir.priority_rows(fsnap, nz[0], nz[1], K, ipa, 1, prefs=prefs, pw=(1, 1), loc=loc,
                                          lw=(1, 10000), spread=spread, w_spread=1)
        np.testing.assert_array_equal(nodes, want_n)
        np.testing.assert_array_equal(scores, want_s)
        # the lane rows are the filter-off rows; the companion counts the nodes that fit but for the filter
        eng.set_interpod_filter(False)
        eng.evaluate()
        np.testing.assert_array_equal(rows, eng.reason_rows())
        np.testing.assert_array_equal(eng.fetch_interpod_reason_rows(), np.zeros_like(comp))
        fit = np.unpackbits(plain.fit_bitmap.view(np.uint8), axis=1, bitorder="little")[:, :snap.nodes.n].astype(bool)
        np.testing.assert_array_equal(comp, fr.companion_rows(v, fit))
        # every node that fits but for the filter counts in exactly one companion bin
        np.testing.assert_array_equal(comp.sum(1), (fit & (v != fr.PASS)).sum(1))
    finally:
        eng.close()
        eng2.close()


def test_many_filter_classes(pkg, oracle):
    # more than 32768 filter classes: each pod its own one-per-host anti-affinity term
    P, N = 33000, 40
    snap = random_snapshot(4242, P=P, N=N, G=200, L=5, case="mixed")
    rng = np.random.default_rng(1)
    topo = np.arange(N, dtype=np.uint32)[None, :]
    bnode = rng.integers(0, N, 1500).astype(np.uint32)
    bcls = rng.integers(0, P, len(bnode)).astype(np.uint32)
    node = (np.array([N], np.uint32), topo, np.zeros(P, np.uint32), bnode, bcls,
            (np.arange(P + 1, dtype=np.uint32), np.arange(P, dtype=np.uint32), np.zeros(P, np.int32), np.ones(P, np.uint8)))
    pods = (np.arange(P, dtype=np.uint32), (np.arange(P + 1, dtype=np.uint32), np.arange(P, dtype=np.uint32),
                                            np.full(P, py.ANTI, np.uint8), np.zeros(P, np.uint8)))
    _check_round(pkg, oracle, snap, (node, pods))


def test_switch_off_is_no_sides(pkg, oracle):
    snap = random_snapshot(515, P=150, N=300, G=20, L=9, case="mixed")
    cols = S.node_interpod_filter(snap, 3)
    outs = []
    for sides in (False, True):
        eng = _engine(pkg, snap, cols if sides else None, on=False, fit_bitmap=True, score=True)
        try:
            res = eng.evaluate()
            outs.append([getattr(res, f).copy() for f in ROUND] + [eng.fit_rows(), eng.score_rows()])
            if sides:   # on, then off again: the parent's outputs once more
                eng.set_interpod_filter(True)
                eng.evaluate()
                eng.set_interpod_filter(False)
                res = eng.evaluate()
                outs.append([getattr(res, f).copy() for f in ROUND] + [eng.fit_rows(), eng.score_rows()])
        finally:
            eng.close()
    for a, b in zip(outs[0], outs[1]):
        np.testing.assert_array_equal(a, b)
    for a, b in zip(outs[0], outs[2]):
        np.testing.assert_array_equal(a, b)


def test_prepass_runs_after_changes_only(pkg, oracle):
    snap = random_snapshot(616, P=120, N=200, G=20, L=5, case="mixed")
    cols = S.node_interpod_filter(snap, 4)
    eng = _engine(pkg, snap, cols)
    try:
        def launches():
            n0 = eng.launch_count()
            eng.evaluate()
            return eng.launch_count() - n0
        first = launches()
        steady = launches()
        assert launches() == steady and first > steady
        eng.upload_interpod_filter(node=cols[0])
        assert launches() > steady
        assert launches() == steady
        eng.upload_interpod_filter(pods=cols[1])
        assert launches() > steady
        assert launches() == steady
        eng.set_interpod_filter(False)
        launches()   # the class fit bits are built again without the filter
        off = launches()
        assert launches() == off == steady   # a steady round with the filter on launches what one without it does
        eng.set_interpod_filter(True)
        assert launches() > steady
        assert launches() == steady
    finally:
        eng.close()


def test_pod_side_reuploads(pkg, oracle):
    # many pod-side uploads and switches on one pod table: each adds (class, filter class) keys to the fit classes,
    # which are compacted when mostly stale; every round stays the filter-off fit ANDed with the restatement
    snap = random_snapshot(919, P=300, N=200, G=40, L=5, case="mixed")
    cols = S.node_interpod_filter(snap, 8)
    pcls, cl = cols[1]
    rng = np.random.default_rng(2)
    eng = _engine(pkg, snap, cols, on=False, fit_bitmap=True)
    try:
        W = (snap.nodes.n + 31) // 32
        eng.evaluate()
        off = eng.fit_rows()[:, :W]
        eng.set_interpod_filter(True)
        for k in range(40):
            pods = (pcls[rng.permutation(len(pcls))], cl)
            eng.upload_interpod_filter(pods=pods)
            if k % 13 == 5:
                eng.set_interpod_filter(False)
                eng.evaluate()
                np.testing.assert_array_equal(eng.fit_rows()[:, :W], off)
                eng.set_interpod_filter(True)
            if k % 4 == 3:
                eng.evaluate()
                v = fr.verdicts((cols[0], pods), snap.nodes.n)
                np.testing.assert_array_equal(eng.fit_rows()[:, :W], off & fr.pack_bits(v == fr.PASS), err_msg=str(k))
    finally:
        eng.close()


def _code(pkg, fn, *a):
    with pytest.raises(pkg.capi.BsError) as ei:
        fn(*a)
    return ei.value.code


def test_drop_rules_and_errors(pkg, oracle):
    capi = pkg.capi
    snap = random_snapshot(717, P=60, N=100, G=10, L=5, case="mixed")
    cols = S.node_interpod_filter(snap, 6)
    eng = _engine(pkg, snap, cols)
    try:
        eng.evaluate()
        eng.upload_nodes(snap.nodes)   # drops the node side
        st = _code(pkg, eng.evaluate)
        eng.upload_interpod_filter(node=cols[0])
        eng.evaluate()
        eng.update_nodes(np.array([0], np.uint32), snap.nodes.take(np.array([0])))   # drops it too
        assert _code(pkg, eng.evaluate) == st
        eng.upload_interpod_filter(node=cols[0])
        eng.upload_pods(snap.pods)     # drops the pod side
        assert _code(pkg, eng.evaluate) == st
        eng.upload_interpod_filter(pods=cols[1])
        eng.evaluate()
        nv, topo, tkey, bnode, bcls, (boff, bterm, bown, bmatch) = cols[0]
        pcls, (poff, pterm, prole, pself) = cols[1]
        bad_node = [
            ((nv, topo, tkey, np.array([snap.nodes.n], np.uint32), np.array([capi.IPF_NONE], np.uint32),
              (boff, bterm, bown, bmatch)), "index"),
            ((nv, topo, tkey, bnode, bcls, (boff, bterm, np.full_like(bown, 2), bmatch)), "range"),
            ((nv, topo[:, :-1], tkey, bnode, bcls, (boff, bterm, bown, bmatch)), "inval"),
        ]
        got = [_code(pkg, eng.upload_interpod_filter, b, None) for b, _ in bad_node]
        assert len(set(got)) == 3
        eng.upload_interpod_filter(node=cols[0])
        bad_pods = [
            (np.full(len(pcls), len(poff), np.uint32), (poff, pterm, prole, pself)),   # class out of range
            (pcls, (poff, pterm, np.full_like(prole, 3), pself)),                     # role
            (pcls, (poff, pterm, prole, np.full_like(pself, 2))),                     # self_match
            (pcls[:-1], (poff, pterm, prole, pself)),                                 # n_pods
        ]
        got = [_code(pkg, eng.upload_interpod_filter, None, b) for b in bad_pods]
        assert got[0] != got[1] and got[2] not in (got[0], got[1]) and got[3] == got[1]
        assert _code(pkg, eng.evaluate) == st   # a failing upload leaves the side dropped
        # a term outside the node side's dictionary
        eng.upload_interpod_filter(pods=(pcls, (poff, np.full_like(pterm, len(tkey)), prole, pself)))
        assert _code(pkg, eng.evaluate) == got[0]
        # the caps: a class longer than BS_IPF_CLASS_MAX entries
        long = (np.zeros(len(pcls), np.uint32), (np.array([0, 65], np.uint32), np.zeros(65, np.uint32),
                                                  np.zeros(65, np.uint8), np.zeros(1, np.uint8)))
        assert _code(pkg, eng.upload_interpod_filter, None, long) == got[1]
    finally:
        eng.close()


def test_refusals(pkg, oracle):
    snap = random_snapshot(818, P=40, N=60, G=8, L=5, case="mixed")
    cols = S.node_interpod_filter(snap, 7)
    eng = _engine(pkg, snap, cols)
    try:
        res = eng.evaluate()
        calls = [lambda: eng.replay(res.order), lambda: eng.replay(res.order, priority=True),
                 lambda: eng.preempt(np.array([0], np.uint32)), lambda: eng.preempt_walk(np.array([0], np.uint32))]
        codes = [_code(pkg, c) for c in calls]
        assert len(set(codes)) == 1
        assert "MatchInterPodAffinity" in eng.lib.bs_last_error(eng.h).decode()
        eng.set_interpod_filter(False)
        eng.replay(res.order)   # with the filter off the walk runs again
    finally:
        eng.close()


def test_cases_on_device(pkg, oracle):
    # the hand-built cases through the engine: one node table per case, every pod fitting every node otherwise
    for name, nodes, existing, pending, answers in cases.CASES:
        N, P = len(nodes), len(pending)
        base = random_snapshot(9, P=P, N=N, G=1, L=5, case="mixed")
        cols = py.pack(nodes, existing, pending)
        v = fr.verdicts(cols, N)
        assert v.tolist() == [[fr.PASS if x == "" else "_EAN".index(x) for x in answers[p.name]] for p in pending]
        eng = _engine(pkg, base, cols, fit_bitmap=True)
        try:
            eng.evaluate()
            fit_on = eng.fit_rows()[:, :1]
            eng.set_interpod_filter(False)
            eng.evaluate()
            fit_off = eng.fit_rows()[:, :1]
        finally:
            eng.close()
        np.testing.assert_array_equal(fit_on, fit_off & fr.pack_bits(v == fr.PASS), err_msg=name)


def test_cfg4_sampled(pkg, oracle):
    snap = S.config(4)
    cols = S.node_interpod_filter(snap, 11)
    rng = np.random.default_rng(3)
    pods = np.sort(rng.choice(np.flatnonzero(cols[1][0] != py.IPF_NONE), 4, replace=False)).astype(np.uint32)
    eng = _engine(pkg, snap, cols, fit_bitmap=True)
    try:
        eng.evaluate()
        on = np.stack([eng.fit_rows(int(p), 1)[0] for p in pods])
        eng.set_interpod_filter(False)
        eng.evaluate()
        off = np.stack([eng.fit_rows(int(p), 1)[0] for p in pods])
    finally:
        eng.close()
    v = fr.verdicts(cols, snap.nodes.n, pods)
    W = (snap.nodes.n + 31) // 32
    np.testing.assert_array_equal(on[:, :W], off[:, :W] & fr.pack_bits(v == fr.PASS))
    assert (v != fr.PASS).any()
