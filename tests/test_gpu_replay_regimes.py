"""GPU: every designed case of tests/replay_regime_cases.py through bs_replay against the oracle's walk and through
bs_replay_priority under two weight sets against its CPU restatement, bit-exact per queue position and on the whole
after-state, each asserting through bs_replay_shape the regime it was built for: the block cache at its limits and
off, 31 / 32 / 33 representative classes, the dead-node skip, findMaxPG buckets past 32 768 groups, the panic, and
the small edges of first-fit bs_replay.  The restatement of bs_replay_priority takes about 2 s per weight set at
1 048 576 nodes on one CPU core, which keeps all three cache-limit cases in; the whole file ran in 37 s on an H100
80GB HBM3 at its 700 W power limit."""
import numpy as np
import pytest

import replay_priority_ref as rpr
import replay_regime_cases as rc
from randsnap import S

pytestmark = pytest.mark.gpu

CASES = rc.cases()
WEIGHTS = [(1, 0, 1), (0, 1, 3)]
AFTER = dict(node_requested=("nodes", "requested"), node_pod_count=("nodes", "pod_count"),
             node_req_present=("nodes", "req_present"), group_matched=("groups", "matched"),
             group_flags=("groups", "flags"), group_min_res=("groups", "min_res"),
             group_min_res_present=("groups", "min_res_present"), group_rep_sel=("groups", "rep_sel"),
             group_rep_tol=("groups", "rep_tol"))


def _same(got, pf, node, ready, after):
    np.testing.assert_array_equal(got["prefilter"], pf)
    np.testing.assert_array_equal(got["node"], node)
    np.testing.assert_array_equal(got["ready"], ready)
    for k, (t, f) in AFTER.items():
        np.testing.assert_array_equal(got[k], getattr(getattr(after, t), f), err_msg=k)


def _regime(eng, case, snap=None, n_queue=None, **over):
    want = rc.regime(case.snap if snap is None else snap, len(case.queue) if n_queue is None else n_queue)
    want.update(case.regime)
    want.update(over)
    got = eng.replay_shape()
    assert {k: got[k] for k in want} == want
    return got


@pytest.mark.parametrize("name", list(CASES))
def test_first_fit(pkg, oracle, name):
    c = CASES[name]
    pf, node, ready, after, at = oracle.replay(c.snap, c.queue, panic=True)
    assert at == c.panic_at
    eng = pkg.Engine(c.snap.lanes)
    try:
        eng.upload(c.snap)
        if at is None:
            _same(eng.replay(c.queue), pf, node, ready, after)
            _regime(eng, c)
            return
        with pytest.raises(pkg.capi.BsError) as ei:
            eng.replay(c.queue)
        assert ei.value.code == pkg.capi.BS_E_REF_PANIC
        _regime(eng, c)
        # the same engine walks a queue without the pod that brings the min_member 0 group into findMaxPG
        q = c.queue[c.snap.pods.gid[c.queue] != 2]
        pf, node, ready, after, at = oracle.replay(c.snap, q, panic=True)
        assert at is None
        _same(eng.replay(q), pf, node, ready, after)
        _regime(eng, c, n_queue=len(q))
    finally:
        eng.close()


@pytest.mark.parametrize("name", [n for n, c in CASES.items() if c.priority])
def test_priority(pkg, oracle, name):
    c = CASES[name]
    node_nz, pod_nz = S.nonzero_requests(c.snap, 3)
    eng = pkg.Engine(c.snap.lanes)
    try:
        eng.upload(c.snap)
        eng.upload_nonzero(node=node_nz, pods=pod_nz)
        for w in WEIGHTS:
            eng.set_score_weights(*w)
            got = eng.replay(c.queue, priority=True)
            pf, node, ready, after, nz_after = rpr.replay_priority(c.snap, node_nz, pod_nz, c.queue, w)
            _same(got, pf, node, ready, after)
            np.testing.assert_array_equal(got["node_nonzero"], nz_after)
            _regime(eng, c)
    finally:
        eng.close()


def test_priority_panics_where_first_fit_does(pkg, oracle):
    c = CASES["panic_panic"]
    node_nz, pod_nz = S.nonzero_requests(c.snap, 3)
    eng = pkg.Engine(c.snap.lanes)
    try:
        eng.upload(c.snap)
        eng.upload_nonzero(node=node_nz, pods=pod_nz)
        with pytest.raises(pkg.capi.BsError) as ei:
            eng.replay(c.queue, priority=True)
        assert ei.value.code == pkg.capi.BS_E_REF_PANIC
        q = c.queue[c.snap.pods.gid[c.queue] != 2]
        got = eng.replay(q, priority=True)
        pf, node, ready, after, nz_after = rpr.replay_priority(c.snap, node_nz, pod_nz, q)
        _same(got, pf, node, ready, after)
        np.testing.assert_array_equal(got["node_nonzero"], nz_after)
    finally:
        eng.close()


def test_shape_needs_a_walk(pkg):
    c = CASES["small_N1_G30"]
    eng = pkg.Engine(c.snap.lanes)
    try:
        eng.upload(c.snap)
        with pytest.raises(pkg.capi.BsError) as ei:
            eng.replay_shape()
        assert ei.value.code == pkg.capi.BS_E_STATE
    finally:
        eng.close()


def test_row_updates_between_walks(pkg, oracle):
    """One engine: the 32-class border case, then a node row update (node 1 gains room), then a group row update
    that gives group 0 a class of its own.  The old class stays in the engine's index, so the second walk has 33
    classes: no fit mask and no block cache."""
    c = CASES["classes_32"]
    snap = c.snap.copy()
    eng = pkg.Engine(snap.lanes)
    try:
        eng.upload(snap)
        _same(eng.replay(c.queue), *oracle.replay(snap, c.queue))
        _regime(eng, c, snap)
        rows = snap.nodes.take([1])
        rows.requested[0, 0] -= 500
        eng.update_nodes(np.array([1]), rows)
        snap.nodes.requested[0, 1] -= 500
        _same(eng.replay(c.queue), *oracle.replay(snap, c.queue))
        _regime(eng, c, snap)
        rows = snap.groups.take([0])
        rows.rep_tol[0] = 2000
        eng.update_groups(np.array([0]), rows)
        snap.groups.rep_tol[0] = 2000
        assert rc.rep_classes(snap) == 32
        _same(eng.replay(c.queue), *oracle.replay(snap, c.queue))
        _regime(eng, c, snap, n_rep=33, fitmask=0, cached=0)
    finally:
        eng.close()
