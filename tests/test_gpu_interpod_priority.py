"""GPU: the InterPodAffinity priority (bs_set_interpod_weight) in the round's priority lists, bit-exact against the CPU
restatement tests/interpod_priority_ref.c: every lane build, list lengths, unaligned sizes, every combination of the
ratio term, the node priorities, the locality priorities and SelectorSpread with IPA on (the shared first sweep);
columns packed from objects; the binary64 pins; the pre-pass under contention and at the caps, re-run after each side
is uploaded and not otherwise; weight 0 is the engine without the columns; the other outputs do not move; the drop
rules; every error code; the walk's refusal; sampled pods at cfg4 size under v1.17's whole default profile."""
import numpy as np
import pytest

import interpod_cases as ic
import interpod_priority_ref as ir
import node_priority_ref as npr
import priority_ref as pr
import ratio_priority_ref as rr
from randsnap import S, random_snapshot

pytestmark = pytest.mark.gpu

PW = (1, 1)
LW = (1, 10000)


def _ratio(L, on):
    return (2, rr.BIN_PACK, [1, 1, 0, 0] + [1] * (L - 4), 1) if on else npr.NO_RATIO


def _engine(pkg, snap, K, nz, interpod, w, ratio=None, prefs=None, loc=None, spread=None, weights=(1, 0, 1), **kw):
    eng = pkg.Engine(snap.lanes, 0, priority_k=K, **kw)
    eng.upload(snap)
    eng.upload_nonzero(node=nz[0], pods=nz[1])
    eng.set_score_weights(*weights)
    if ratio is not None and ratio[0]:
        eng.set_ratio_priority(*ratio)
    if prefs is not None:
        eng.upload_preferences(node=(prefs[0], prefs[1]), pods=(prefs[2], prefs[3]))
        eng.set_node_priority_weights(*PW)
    if loc is not None:
        eng.upload_locality(node=loc[0], pods=loc[1])
        eng.set_locality_weights(*LW)
    if spread is not None:
        eng.upload_spread(node=spread[0], pods=spread[1])
        eng.set_spread_weight(1)
    if interpod is not None:
        eng.upload_interpod(node=interpod[0], pods=interpod[1])
    eng.set_interpod_weight(w)
    return eng


def _check(pkg, snap, K, w, seed, ratio_on=False, pref_on=False, loc_on=False, spread_on=False, weights=(1, 0, 1),
           interpod=None):
    nz = S.nonzero_requests(snap, seed)
    interpod = S.node_interpod(snap, seed) if interpod is None else interpod
    prefs = S.node_preferences(snap, seed) if pref_on else None
    loc = S.node_locality(snap, seed) if loc_on else None
    spread = S.node_spread(snap, seed) if spread_on else None
    ratio = _ratio(snap.lanes, ratio_on)
    eng = _engine(pkg, snap, K, nz, interpod, w, ratio, prefs, loc, spread, weights)
    try:
        eng.evaluate()
        nodes, scores = eng.priority_rows()
    finally:
        eng.close()
    want_n, want_s = ir.priority_rows(snap, nz[0], nz[1], K, interpod, w, ratio, weights, prefs,
                                      PW if pref_on else (0, 0), loc, LW if loc_on else (0, 0), spread,
                                      1 if spread_on else 0)
    np.testing.assert_array_equal(nodes, want_n)
    np.testing.assert_array_equal(scores, want_s)
    return nodes, scores


@pytest.mark.parametrize("L", [5, 9, 16])
@pytest.mark.parametrize("ratio_on", [False, True])
@pytest.mark.parametrize("pref_on", [False, True])
@pytest.mark.parametrize("loc_on", [False, True])
@pytest.mark.parametrize("spread_on", [False, True])
def test_flag_combinations(pkg, oracle, L, ratio_on, pref_on, loc_on, spread_on):
    snap = random_snapshot(3100 + L, P=200, N=500, G=30, L=L, case="mixed")
    K = {5: 1, 9: 7, 16: 32}[L]
    _check(pkg, snap, K, 1, L, ratio_on, pref_on, loc_on, spread_on)


@pytest.mark.parametrize("K", [1, 7, 32])
@pytest.mark.parametrize("w", [1, 7])
def test_lengths_and_weights(pkg, oracle, K, w):
    snap = random_snapshot(3150 + K, P=300, N=900, G=30, L=6, aff=3)
    _check(pkg, snap, K, w, K, K == 7, K == 32, weights=(2, 1, 3))


@pytest.mark.parametrize("P,N", [(1, 1), (37, 31), (70, 33), (131, 511), (95, 1025)])
def test_unaligned_sizes(pkg, oracle, P, N):
    snap = random_snapshot(P * 5 + N + 3100, P=P, N=N, G=9, L=6)
    _check(pkg, snap, 7, 1, N, N % 2 == 1)


@pytest.mark.parametrize("seed", range(3))
def test_columns_packed_from_objects(pkg, oracle, seed):
    snap = random_snapshot(3160 + seed, P=120, N=200, G=20, L=5)
    pending, bound, labels = ic.random_objects(seed, snap.nodes.n, snap.pods.n, invalid=0.02 * seed)
    _check(pkg, snap, 16, 1, seed, interpod=ic.columns(pending, bound, labels, hard=[1, 0, 100][seed]))


def _pins_case(raws, at, N, P, p):
    """One hostname key and two terms: bound class 0 matches term 0, bound class 1 term 1, and pod p's class owns +1
    on term 0 and -1 on term 1, so its raw on node n is (class-0 pods on n) - (class-1 pods on n): raws[k] on node
    at[k], 0 elsewhere (which moves neither extreme: both start at 0)."""
    bnode, bcls = [], []
    for n, r in zip(at, raws):
        bnode += [n] * abs(r)
        bcls += [0 if r > 0 else 1] * abs(r)
    bcl = ([0, 1, 2], [0, 1], [0, 0], [1, 1])
    pcl = ([0, 2], [0, 1], [1, -1], [0, 0])
    pcls = np.full(P, S.IPA_NONE, np.uint32)
    pcls[p] = 0
    return ([N], [np.arange(N)], [0, 0], bnode, bcls, bcl), (pcls, pcl)


PINS = {(-7, 22, 43): [0, 57, 100], (10, 20, 0): [50, 100, 0], (-10, -20, 0): [50, 0, 100], (0, 0, 0): [0, 0, 0]}


def test_binary64_pins(pkg, oracle):
    """Raws -7, 22, 43 give 0, 57 (not 58), 100; 10, 20, 0 give 50, 100, 0 (min stays 0); -10, -20, 0 give 50, 0,
    100 (max stays 0); all 0 give 0."""
    snap = random_snapshot(3170, P=40, N=60, G=4, L=5)
    zero = ([1], [np.zeros(snap.nodes.n)], [0], [], [], ([0], [], [], [])), (np.full(snap.pods.n, S.IPA_NONE), ([0], [], [], []))
    fit = ir.ipa_matrix(snap, zero) >= 0
    p = int(np.argmax(fit.sum(axis=1)))
    at = np.nonzero(fit[p])[0][:3]
    assert len(at) == 3
    for raws, ipa in PINS.items():
        interpod = _pins_case(raws, at, snap.nodes.n, snap.pods.n, p)
        assert ir.raw_matrix(interpod, snap.nodes.n, [p])[0][at].tolist() == list(raws)
        assert ir.ipa_matrix(snap, interpod, [p])[0][at].tolist() == ipa
        _check(pkg, snap, 32, 1, 1, interpod=interpod)
        _check(pkg, snap, 32, 5, 1, True, True, interpod=interpod)


def test_prepass_contention_and_caps(pkg, oracle):
    """Every bound pod in one zone value (one M / S slot per term takes every atomic), 2^16 own weights and classes of
    BS_IPA_CLASS_MAX entries."""
    snap = random_snapshot(3180, P=150, N=400, G=20, L=5)
    N = snap.nodes.n
    rng = np.random.default_rng(3)
    T = 64
    n_values, topo, term_key = [1], [[0] * N], [0] * T
    own = rng.choice([-(1 << 16), 1 << 16, 3, -5], T).astype(np.int32)
    bcl = ([0, T], np.arange(T), own, np.ones(T, np.uint8))
    pcl = ([0, T, 2 * T], np.r_[np.arange(T), np.arange(T)], np.r_[own, -own], np.r_[np.ones(T), np.zeros(T)])
    V = 50_000
    interpod = ((n_values, topo, term_key, rng.integers(0, N, V), np.zeros(V, np.uint32), bcl),
                (rng.integers(0, 2, snap.pods.n).astype(np.uint32), pcl))
    _check(pkg, snap, 8, 1, 2, interpod=interpod)
    # and spread over the hostname key: each node's own slot
    interpod2 = (([N], [np.arange(N)], term_key, *interpod[0][3:]), interpod[1])
    _check(pkg, snap, 8, 3, 2, interpod=interpod2)


def test_prepass_runs_after_each_side_changes_and_not_otherwise(pkg, oracle):
    snap = random_snapshot(3190, P=200, N=500, G=20, L=6)
    nz = S.nonzero_requests(snap, 4)
    node, pods = S.node_interpod(snap, 4)
    eng = _engine(pkg, snap, 16, nz, (node, pods), 0)
    try:
        def launches():
            n0 = eng.launch_count()
            eng.evaluate()
            return eng.launch_count() - n0
        launches()
        base = launches()   # weight 0: the kernel without IPA and no pre-pass
        eng.set_interpod_weight(1)
        assert launches() == base + 2   # the mass and the class kernel ahead of the IPA kernel
        assert launches() == base
        eng.upload_interpod(pods=pods)
        assert launches() == base + 1   # the class kernel alone: M and S did not change
        eng.upload_interpod(node=node)
        assert launches() == base + 2
        eng.set_interpod_weight(0)
        eng.upload_interpod(node=node)
        assert launches() == base
        eng.set_interpod_weight(1)
        assert launches() == base + 2   # built at the first evaluation that reads it
        eng.evaluate()
        nodes, scores = eng.priority_rows()
    finally:
        eng.close()
    want_n, want_s = ir.priority_rows(snap, nz[0], nz[1], 16, (node, pods), 1)
    np.testing.assert_array_equal(nodes, want_n)
    np.testing.assert_array_equal(scores, want_s)


def test_zero_weight_is_the_engine_without_columns(pkg, oracle):
    snap = random_snapshot(3200, P=300, N=800, G=30, L=6, aff=2)
    nz = S.nonzero_requests(snap, 3200)
    interpod = S.node_interpod(snap, 3200)
    out = []
    for with_cols in (False, True):
        eng = _engine(pkg, snap, 9, nz, interpod if with_cols else None, 0)
        try:
            eng.evaluate()
            out.append(eng.priority_rows())
            if with_cols:   # on, then off again on the same engine
                eng.set_interpod_weight(1)
                eng.evaluate()
                on = eng.priority_rows()
                eng.set_interpod_weight(0)
                eng.evaluate()
                out.append(eng.priority_rows())
        finally:
            eng.close()
    for nodes, scores in out[1:]:
        np.testing.assert_array_equal(nodes, out[0][0])
        np.testing.assert_array_equal(scores, out[0][1])
    assert not np.array_equal(on[1], out[0][1])
    n0, s0 = pr.priority_rows(snap, nz[0], nz[1], 9)
    np.testing.assert_array_equal(out[0][0], n0)
    np.testing.assert_array_equal(out[0][1], s0)


def test_other_outputs_do_not_move(pkg, oracle):
    snap = random_snapshot(3201, P=300, N=800, G=30, L=6)
    nz = S.nonzero_requests(snap, 3201)
    interpod = S.node_interpod(snap, 3201)
    got = []
    for w in (0, 3):
        eng = _engine(pkg, snap, 8, nz, interpod, w, fit_bitmap=True, topk=8, reasons=True)
        try:
            res = eng.evaluate()
            got.append((res, eng.fit_rows(), eng.topk_rows(), eng.reason_rows()))
        finally:
            eng.close()
    (r0, f0, t0, q0), (r1, f1, t1, q1) = got
    for f in ("prefilter", "feasible_count", "best_node", "best_score", "admit", "order", "rank"):
        np.testing.assert_array_equal(getattr(r0, f), getattr(r1, f), err_msg=f)
    np.testing.assert_array_equal(f0, f1)
    np.testing.assert_array_equal(t0[0], t1[0])
    np.testing.assert_array_equal(t0[1], t1[1])
    np.testing.assert_array_equal(q0, q1)


def test_drop_rules(pkg, oracle):
    """bs_update_nodes drops the node side, bs_upload_pods the pod side; uploading them again restores the lists."""
    c = pkg.capi
    snap = random_snapshot(3202, P=200, N=500, G=20, L=6)
    nz = S.nonzero_requests(snap, 3202)
    node, pods = S.node_interpod(snap, 3202)
    eng = _engine(pkg, snap, 16, nz, (node, pods), 1)
    try:
        eng.evaluate()
        idx = np.arange(0, snap.nodes.n, 7)
        eng.update_nodes(idx, snap.nodes.take(idx))
        eng.upload_nonzero(node=nz[0])
        with pytest.raises(c.BsError) as ei:
            eng.evaluate()
        assert ei.value.code == c.BS_E_STATE
        node2 = node[:3] + (np.r_[node[3], idx].astype(np.uint32), np.r_[node[4], np.zeros(len(idx), np.uint32)],
                            node[5])   # pods bound on the changed nodes
        eng.upload_interpod(node=node2)
        eng.evaluate()
        nodes, scores = eng.priority_rows()
        eng.upload(snap)   # the pod table again: both sides go
        eng.upload_nonzero(node=nz[0], pods=nz[1])
        eng.upload_interpod(node=node2)
        with pytest.raises(c.BsError) as ei:
            eng.evaluate()
        assert ei.value.code == c.BS_E_STATE
        eng.upload_interpod(pods=pods)
        eng.evaluate()
        nodes2, scores2 = eng.priority_rows()
    finally:
        eng.close()
    want_n, want_s = ir.priority_rows(snap, nz[0], nz[1], 16, (node2, pods), 1)
    for n, s in ((nodes, scores), (nodes2, scores2)):
        np.testing.assert_array_equal(n, want_n)
        np.testing.assert_array_equal(s, want_s)


def test_errors_and_the_walk(pkg):
    c = pkg.capi
    snap = random_snapshot(3210, P=50, N=80, G=5, L=6)
    nz = S.nonzero_requests(snap, 3210)
    node, pods = S.node_interpod(snap, 3210)
    nv, topo, tkey, bnode, bcls, bcl = node
    pcls, pcl = pods
    N = snap.nodes.n

    def code(f, *a, **kw):
        with pytest.raises(c.BsError) as ei:
            f(*a, **kw)
        return ei.value.code

    def with_node(**kw):
        d = dict(nv=nv, topo=topo, tkey=tkey, bnode=bnode, bcls=bcls, bcl=bcl)
        d.update(kw)
        return (d["nv"], d["topo"], d["tkey"], d["bnode"], d["bcls"], d["bcl"])

    def cl_with(cl, k, v, i=0):
        cl = [np.array(x).copy() for x in cl]
        cl[k][i] = v
        return tuple(cl)

    eng = _engine(pkg, snap, 4, nz, None, 0)
    try:
        eng.evaluate()
        eng.replay(priority=True)
        # wrong sizes, too many keys or bound pods, malformed class tables: BS_E_INVAL
        assert code(eng.upload_interpod, node=with_node(topo=np.asarray(topo)[:, :-1])) == c.BS_E_INVAL
        assert code(eng.upload_interpod, pods=(pcls[:-1], pcl)) == c.BS_E_INVAL
        assert code(eng.upload_interpod, node=with_node(nv=np.ones(65, np.uint32), topo=np.zeros((65, N)))) == c.BS_E_INVAL
        big = np.zeros(c.IPA_BOUND_MAX + 1, np.uint32)
        assert code(eng.upload_interpod, node=with_node(bnode=big, bcls=big + c.IPA_NONE)) == c.BS_E_INVAL
        assert code(eng.upload_interpod, node=with_node(bcl=cl_with(bcl, 0, 1))) == c.BS_E_INVAL   # offset[0] != 0
        wide = (np.array([0, 65], np.uint32), np.arange(65), np.ones(65, np.int32), np.ones(65, np.uint8))
        none = np.full(len(bcls), c.IPA_NONE, np.uint32)
        assert code(eng.upload_interpod, node=with_node(tkey=np.zeros(65, np.uint32), bcl=wide, bcls=none)) == c.BS_E_INVAL
        twice = (np.array([0, 2], np.uint32), np.array([1, 1]), np.ones(2, np.int32), np.ones(2, np.uint8))
        assert code(eng.upload_interpod, pods=(np.zeros(len(pcls), np.uint32), twice)) == c.BS_E_INVAL
        huge_nv = np.array([c.IPA_TERM_MAX_BYTES // 16 + 1], np.uint32)
        assert code(eng.upload_interpod, node=with_node(nv=huge_nv, topo=np.zeros((1, N)), tkey=[0],
                                                        bcl=([0], [], [], []), bcls=none)) == c.BS_E_INVAL
        n_cls = c.IPA_TABLE_MAX_BYTES // (((N + 31) // 32) * 32 * 8) + 1
        many = (np.zeros(n_cls + 1, np.uint32), [], [], [])
        assert code(eng.upload_interpod, pods=(np.full(len(pcls), c.IPA_NONE, np.uint32), many)) == c.BS_E_INVAL
        # ids out of range: BS_E_INDEX; own and match out of range: BS_E_RANGE
        bad_topo = np.array(topo).copy()
        bad_topo[1, 3] = nv[1]
        assert code(eng.upload_interpod, node=with_node(topo=bad_topo)) == c.BS_E_INDEX
        assert code(eng.upload_interpod, node=with_node(tkey=np.r_[tkey[:-1], len(nv)])) == c.BS_E_INDEX
        assert code(eng.upload_interpod, node=with_node(bnode=np.r_[bnode[:-1], N])) == c.BS_E_INDEX
        assert code(eng.upload_interpod, node=with_node(bcls=np.r_[bcls[:-1], len(bcl[0]) - 1])) == c.BS_E_INDEX
        assert code(eng.upload_interpod, node=with_node(bcl=cl_with(bcl, 1, len(tkey)))) == c.BS_E_INDEX
        assert code(eng.upload_interpod, pods=(np.r_[pcls[:-1], len(pcl[0]) - 1], pcl)) == c.BS_E_INDEX
        for v in (-(1 << 16) - 1, (1 << 16) + 1):
            assert code(eng.upload_interpod, node=with_node(bcl=cl_with(bcl, 2, v))) == c.BS_E_RANGE
            assert code(eng.upload_interpod, pods=(pcls, cl_with(pcl, 2, v))) == c.BS_E_RANGE
        assert code(eng.upload_interpod, node=with_node(bcl=cl_with(bcl, 3, 2))) == c.BS_E_RANGE
        assert code(eng.upload_interpod, pods=(pcls, cl_with(pcl, 3, 2))) == c.BS_E_RANGE
        eng.upload_interpod(node=with_node(bcl=cl_with(bcl, 2, 1 << 16)))
        # missing sides: BS_E_STATE before anything launches, only while the weight is non-zero
        eng.evaluate()
        eng.set_interpod_weight(1)
        assert code(eng.evaluate) == c.BS_E_STATE    # no pod side yet
        eng.upload_interpod(pods=pods)
        eng.evaluate()
        assert code(eng.upload_interpod, node=with_node(topo=np.asarray(topo)[:, :-1])) == c.BS_E_INVAL
        assert code(eng.evaluate) == c.BS_E_STATE    # the failing call dropped the node side
        eng.upload_interpod(node=node)
        eng.evaluate()
        assert code(eng.upload_interpod, pods=(pcls, cl_with(pcl, 3, 2))) == c.BS_E_RANGE
        assert code(eng.evaluate) == c.BS_E_STATE    # ... and the pod side
        # a pod class's term at or above the node side's n_terms: BS_E_INDEX at evaluation
        eng.upload_interpod(pods=(pcls, cl_with(pcl, 1, len(tkey))))
        assert code(eng.evaluate) == c.BS_E_INDEX
        eng.set_interpod_weight(0)
        eng.evaluate()
        eng.set_interpod_weight(1)
        eng.upload_interpod(pods=pods)
        # the walk refuses a non-zero weight and runs again at 0
        assert code(lambda: eng.replay(priority=True)) == c.BS_E_INVAL
        eng.set_interpod_weight(0)
        eng.replay(priority=True)
    finally:
        eng.close()


def test_full_size_cfg4_default_profile(pkg, oracle, snapshot_mod):
    """cfg4 under v1.17's whole default profile: resource weights (1, 0, 1), TaintToleration / NodeAffinity (1, 1),
    ImageLocality / NodePreferAvoidPods (1, 10000), SelectorSpread 1 and InterPodAffinity 1 with hard weight 1."""
    snap = snapshot_mod.config(4)
    nz = snapshot_mod.nonzero_requests(snap, 4)
    interpod = snapshot_mod.node_interpod(snap, 4, n_bound=300_000, hard=1)
    prefs = snapshot_mod.node_preferences(snap, 4)
    loc = snapshot_mod.node_locality(snap, 4)
    spread = snapshot_mod.node_spread(snap, 4, n_zones=8, n_classes=32)
    eng = _engine(pkg, snap, 16, nz, interpod, 1, prefs=prefs, loc=loc, spread=spread, fit_bitmap=False)
    try:
        res = eng.evaluate()
        nodes, scores = eng.priority_rows()
    finally:
        eng.close()
    idx = np.sort(np.random.default_rng(4).choice(snap.pods.n, 100, replace=False))
    want_n, want_s = ir.priority_rows(snap, nz[0], nz[1], 16, interpod, 1, prefs=prefs, pw=PW, loc=loc, lw=LW,
                                      spread=spread, w_spread=1, pods=idx)
    np.testing.assert_array_equal(nodes[idx], want_n)
    np.testing.assert_array_equal(scores[idx], want_s)
    np.testing.assert_array_equal((nodes >= 0).sum(axis=1), np.minimum(16, res.feasible_count))


def test_plugin_inter_pod_affinity_weight():
    """The C++ plugin's SetInterPodAffinityWeight(1) over objects: PriorityNodes equals an engine called directly with
    PackInterPodAffinity's columns, and ReplayQueue(kPriority) refuses the weight."""
    import json
    import subprocess

    import native
    o = json.loads(subprocess.check_output([native.cpp_program("plugin_interpod_priority_test"), "gpu"], text=True))
    sc = o["scenarios"][0]
    assert sc["plugin"] == sc["engine"]
    assert sc["replay_refused"]
    assert any(len(row) for row in sc["plugin"])
