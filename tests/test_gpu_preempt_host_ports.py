"""GPU: bs_preempt and bs_preempt_walk under the PodFitsHostPorts filter, bit-exact against the CPU restatement
tests/preempt_host_ports_ref.c (node, n_victims, n_candidates, offsets, victims in order, and for the walk outcome and
evicted_by, with and without BS_PREEMPT_GANG): the designed cases of tests/preempt_host_ports_cases.py, random tables
at every register width of the kernels (MAXL 5, 9 and 16), the filter off with the bound side uploaded, all-zero row
masks, every refusal and drop of the bound side, and one long-lived engine through uploads, node updates, switch flips,
preemptions and walks."""
import importlib
import itertools

import numpy as np
import pytest

import host_ports_ref
import preempt_host_ports_cases as H
import preempt_host_ports_ref as R
import preempt_walk_cases as W

S = importlib.import_module("batch-scheduler_b200.snapshot")
E = importlib.import_module("batch-scheduler_b200.engine")
capi = importlib.import_module("batch-scheduler_b200.capi")

pytestmark = pytest.mark.gpu


def _engine(snap, bound, cols, ports, on=True):
    eng = E.Engine(snap.lanes)
    eng.upload(snap)
    eng.upload_bound_pods(bound)
    eng.upload_host_ports(node=cols[0], pods=cols[1])
    if ports is not None:
        eng.upload_bound_host_ports(ports)
    eng.set_host_port_filter(on)
    return eng


def _same(got, want, walk=False):
    for f in ("node", "n_victims", "n_candidates", "victim_offset", "victims") + (("outcome", "evicted_by") if walk else ()):
        np.testing.assert_array_equal(getattr(got, f), getattr(want, f), err_msg=f)


def _code(fn, *a):
    with pytest.raises(capi.BsError) as ei:
        fn(*a)
    return ei.value.code


def _check_all(eng, snap, bound, cols, ports, pods_walk, gangs=(False, True)):
    """bs_preempt over every pod and the walk over `pods_walk`, against the restatement; returns the walk results."""
    _same(eng.preempt(np.arange(snap.pods.n, dtype=np.uint32)), R.preempt(snap, bound, cols, ports))
    out = []
    for gang in gangs:
        got = eng.preempt_walk(np.asarray(pods_walk, np.uint32), gang=gang)
        _same(got, R.walk(snap, bound, cols, ports, pods_walk, gang), walk=True)
        out.append(got)
    return out


def random_case(seed, L, violating=0.3, P=64, N=90, G=10, p_hold=0.6):
    """A random table with the filter's columns.  W.queue(gang=True) gives each group one priority, which it does to
    the snapshot in place: it runs here, before any engine sees the table (later calls change nothing)."""
    snap, bound = W.random_table(seed, L, violating, P=P, N=N, G=G, max_per_node=12)
    W.queue(snap, gang=True)
    (entries, used), want = host_ports_ref.random_columns(snap, seed, n_entries=6, grouped=0.6, node_bits=3)
    rng = np.random.default_rng(seed + 7)
    for p in range(P):
        if want[p] == 0 and rng.random() < 0.8:
            want[p] = np.uint64(1) << np.uint64(rng.integers(0, len(entries)))
    return snap, bound, ((entries, used), want), R.random_bound_ports(snap, bound, used, seed, p_hold)


@pytest.mark.parametrize("name", sorted(H.cases()))
def test_designed_case(name):
    snap, bound, cols, ports, pods, walk, gang, want = H.cases()[name]
    eng = _engine(snap, bound, cols, ports)
    try:
        if walk:
            got = eng.preempt_walk(np.asarray(pods, np.uint32), gang=gang)
            _same(got, R.walk(snap, bound, cols, ports, pods, gang), walk=True)
            assert [(int(got.node[k]), got.victims_of(k), int(got.n_candidates[k]), int(got.outcome[k]))
                    for k in range(len(pods))] == want
            other = eng.preempt_walk(np.asarray(pods, np.uint32), gang=not gang)
            _same(other, R.walk(snap, bound, cols, ports, pods, not gang), walk=True)
        else:
            got = eng.preempt(np.asarray(pods, np.uint32))
            _same(got, R.preempt(snap, bound, cols, ports, pods))
            assert [(int(got.node[k]), got.victims_of(k), int(got.n_candidates[k])) for k in range(len(pods))] == want
            for gang in (False, True):
                q = W.queue(snap, pods, gang=False)
                _same(eng.preempt_walk(np.asarray(q, np.uint32), gang=gang), R.walk(snap, bound, cols, ports, q, gang),
                      walk=True)
    finally:
        eng.close()


@pytest.mark.parametrize("seed,L", list(itertools.product((0, 2, 4), (5, 9, 16))))
def test_random(seed, L):
    """L 5, 9 and 16 run the MAXL 5, 9 and 16 builds of the node, emit and commit kernels with the filter."""
    snap, bound, cols, ports = random_case(seed, L)
    eng = _engine(snap, bound, cols, ports)
    try:
        plain, gang = _check_all(eng, snap, bound, cols, ports, W.queue(snap, gang=True))
        assert len(plain.victims) > 0
    finally:
        eng.close()


def test_filter_off_reads_no_bound_side():
    snap, bound, cols, ports = random_case(11, 5)
    pods = W.queue(snap, gang=True)
    with_side = _engine(snap, bound, cols, ports, on=False)
    without = _engine(snap, bound, cols, None, on=False)
    try:
        _same(with_side.preempt(np.arange(snap.pods.n)), without.preempt(np.arange(snap.pods.n)))
        for gang in (False, True):
            _same(with_side.preempt_walk(pods, gang=gang), without.preempt_walk(pods, gang=gang), walk=True)
    finally:
        with_side.close()
        without.close()


def test_zero_row_masks_free_nothing():
    """With every row mask 0 no eviction frees a port: the answers are the restatement's with no row holding any."""
    snap, bound, cols, _ = random_case(12, 5)
    zero = np.zeros(bound.n, np.uint64)
    eng = _engine(snap, bound, cols, zero)
    try:
        _check_all(eng, snap, bound, cols, zero, W.queue(snap, gang=True))
    finally:
        eng.close()


def test_refusals_and_drops():
    snap, bound, cols, ports = random_case(13, 5, P=20, N=20)
    (entries, used), want = cols
    K = len(entries)
    one = np.array([0], np.uint32)
    calls = (lambda: E.Engine.preempt(eng, one), lambda: E.Engine.preempt_walk(eng, one))
    eng = _engine(snap, bound, cols, None)
    try:
        # no bound side: today's refusal, naming the upload
        for c in calls:
            assert _code(c) == capi.BS_E_INVAL
            msg = eng.lib.bs_last_error(eng.h).decode()
            assert "PodFitsHostPorts" in msg and "bs_upload_bound_host_ports" in msg
        # the upload's own errors, each leaving the side dropped
        assert _code(eng.upload_bound_host_ports, ports[:-1]) == capi.BS_E_INVAL
        assert _code(calls[0]) == capi.BS_E_INVAL
        eng.upload_bound_host_ports(ports)
        eng.preempt(one)
        # MatchInterPodAffinity's refusal comes first
        eng.set_interpod_filter(True)
        for c in calls:
            assert _code(c) == capi.BS_E_INVAL
            assert "MatchInterPodAffinity" in eng.lib.bs_last_error(eng.h).decode()
        eng.set_interpod_filter(False)
        # bits checked when a preemption starts: past n_entries, and outside the row's node's used mask
        bad = ports.copy()
        bad[0] |= np.uint64(1) << np.uint64(K)
        eng.upload_bound_host_ports(bad)
        assert [_code(c) for c in calls] == [capi.BS_E_INDEX] * 2
        outside = ~used[int(bound.node[0])] & np.uint64((1 << K) - 1)
        assert outside != 0
        bad = ports.copy()
        bad[0] |= outside & (~outside + np.uint64(1))   # its lowest bit
        eng.upload_bound_host_ports(bad)
        assert [_code(c) for c in calls] == [capi.BS_E_INVAL] * 2
        # the same bits are fine with the filter off (the side is not read) and again with a node side that uses them
        eng.set_host_port_filter(False)
        eng.preempt(one)
        eng.set_host_port_filter(True)
        wide = used.copy()
        wide[int(bound.node[0])] |= outside
        eng.upload_host_ports(node=(entries, wide))
        eng.preempt(one)
        eng.upload_bound_host_ports(ports)
        # the other sides as a round needs them
        eng.upload_host_ports(pods=want | (np.uint64(1) << np.uint64(K)))
        assert [_code(c) for c in calls] == [capi.BS_E_INDEX] * 2
        eng.upload_host_ports(pods=want, node=cols[0])
        eng.preempt(one)
        eng.upload_pods(snap.pods)   # drops the pod side
        assert [_code(c) for c in calls] == [capi.BS_E_STATE] * 2
        eng.upload_host_ports(pods=want)
        eng.preempt(one)
        # every call that drops the bound table drops the side
        eng.upload_bound_pods(bound)
        assert _code(calls[0]) == capi.BS_E_INVAL
        eng.upload_bound_host_ports(ports)
        eng.upload_groups(snap.groups)
        assert _code(eng.upload_bound_host_ports, ports) == capi.BS_E_STATE
        eng.upload_bound_pods(bound)
        assert _code(calls[0]) == capi.BS_E_INVAL
        eng.upload_bound_host_ports(ports)
        eng.update_nodes(np.array([0], np.uint32), snap.nodes.take([0]))
        eng.upload_bound_pods(bound)
        eng.upload_host_ports(node=cols[0])
        assert _code(calls[0]) == capi.BS_E_INVAL
        eng.upload_bound_host_ports(ports)
        eng.upload_nodes(snap.nodes)
        assert _code(eng.upload_bound_host_ports, ports) == capi.BS_E_STATE
    finally:
        eng.close()


def test_long_lived_engine():
    """One engine through random table uploads, node-row updates, node-side changes, bound-table and bound-side
    uploads, switch flips, preemptions and walks; each answer against the restatement of the state the engine holds."""
    rng = np.random.default_rng(5)
    snap, bound, cols, ports = random_case(21, 5)
    eng = _engine(snap, bound, cols, ports)
    on, have_side = True, True
    checked = updates = 0
    try:
        for step in range(28):
            op = 5 if step % 7 == 6 else rng.integers(0, 6)
            if op == 0:   # a new table and all its sides, into the same engine
                snap, bound, cols, ports = random_case(int(rng.integers(0, 1000)), 5)
                eng.upload(snap)
                eng.upload_bound_pods(bound)
                eng.upload_host_ports(node=cols[0], pods=cols[1])
                eng.upload_bound_host_ports(ports)
                have_side = True
            elif op == 1:   # fresh bound-side masks
                ports = R.random_bound_ports(snap, bound, cols[0][1], int(rng.integers(0, 1000)), rng.random())
                eng.upload_bound_host_ports(ports)
                have_side = True
            elif op == 2:   # a new node side whose used masks grow: the bound side stays valid
                (entries, used), want = cols
                used = used | np.uint64(rng.integers(0, 1 << len(entries)))
                cols = ((entries, used), want)
                eng.upload_host_ports(node=cols[0])
            elif op == 3:
                on = not on
                eng.set_host_port_filter(on)
            elif op == 4:   # the bound table again: the side goes with the old one
                eng.upload_bound_pods(bound)
                have_side = False
                if rng.random() < 0.7:
                    eng.upload_bound_host_ports(ports)
                    have_side = True
            else:   # bs_update_nodes on a few rows (new cpu capacity), which drops the bound table and the node side
                idx = np.unique(rng.integers(0, snap.nodes.n, 4)).astype(np.uint32)
                snap.nodes.alloc[0, idx] += rng.integers(0, 3000, len(idx))
                eng.update_nodes(idx, snap.nodes.take(idx))
                assert _code(eng.upload_bound_host_ports, ports) == capi.BS_E_STATE
                eng.upload_bound_pods(bound)
                eng.upload_host_ports(node=cols[0])
                have_side = rng.random() < 0.7
                if have_side:
                    eng.upload_bound_host_ports(ports)
                updates += 1
            pods = W.queue(snap, gang=True)
            if on and not have_side:
                assert _code(eng.preempt, pods) == capi.BS_E_INVAL
                continue
            if on:
                _check_all(eng, snap, bound, cols, ports, pods, gangs=(bool(step % 2),))
            else:
                import preempt_pdb_ref
                import preempt_walk_ref
                _same(eng.preempt(np.arange(snap.pods.n)), preempt_pdb_ref.preempt(snap, bound))
                _same(eng.preempt_walk(pods, gang=True), preempt_walk_ref.walk(snap, bound, pods, True), walk=True)
            checked += 1
        assert checked >= 12 and updates >= 2
    finally:
        eng.close()
