"""CPU: the restatements of preemption under the PodFitsHostPorts filter.  tests/preempt_host_ports_ref.c and
tests/pyref_preempt_host_ports.py agree on random tables, single-pod and walked, with and without gang units; with no
ports anywhere the C restatement gives tests/preempt_pdb_ref.c's and tests/preempt_walk_ref.c's answers; and the
designed cases of tests/preempt_host_ports_cases.py give their written-out answers."""
import numpy as np
import pytest

import host_ports_ref
import preempt_host_ports_cases as H
import preempt_host_ports_ref as R
import preempt_pdb_ref
import preempt_walk_cases as W
import preempt_walk_ref
import pyref_preempt_host_ports as PY


def random_case(seed, L=5, violating=0.3, P=24, N=12, G=4, p_hold=0.6):
    """A preemption table with the filter's columns: random_columns over it, each bound row holding a random subset of
    its node's used entries, and most preemptors wanting an entry."""
    snap, bound = W.random_table(seed, L, violating, P=P, N=N, G=G, max_per_node=6)
    (entries, used), want = host_ports_ref.random_columns(snap, seed, n_entries=6, grouped=0.6, node_bits=3)
    rng = np.random.default_rng(seed + 7)
    K = len(entries)
    for p in range(P):
        if want[p] == 0 and rng.random() < 0.8:
            want[p] = np.uint64(1) << np.uint64(rng.integers(0, K))
    ports = R.random_bound_ports(snap, bound, used, seed, p_hold)
    return snap, bound, ((entries, used), want), ports


def _as_list(res, walk=False):
    rows = []
    for k in range(len(res.node)):
        r = (int(res.node[k]), res.victims_of(k), int(res.n_candidates[k]))
        rows.append(r + (int(res.outcome[k]),) if walk else r)
    return rows


@pytest.mark.parametrize("name", sorted(H.cases()))
def test_designed_case(name):
    snap, bound, cols, ports, pods, walk, gang, want = H.cases()[name]
    if walk:
        got = R.walk(snap, bound, cols, ports, pods, gang)
        assert _as_list(got, True) == want
        py, evby = PY.walk(snap, bound, cols, ports, pods, gang)
        assert [tuple(r) for r in py] == want and list(got.evicted_by) == evby
    else:
        assert _as_list(R.preempt(snap, bound, cols, ports, pods)) == want
        assert [tuple(r) for r in PY.preempt(snap, bound, cols, ports, pods)] == want


@pytest.mark.parametrize("seed", range(6))
def test_c_and_python_agree(seed):
    snap, bound, cols, ports = random_case(seed)
    got = R.preempt(snap, bound, cols, ports)
    assert _as_list(got) == [tuple(r) for r in PY.preempt(snap, bound, cols, ports, range(snap.pods.n))]
    for gang in (False, True):
        pods = W.queue(snap, gang=gang)
        got = R.walk(snap, bound, cols, ports, pods, gang)
        py, evby = PY.walk(snap, bound, cols, ports, pods, gang)
        assert _as_list(got, True) == [tuple(r) for r in py] and list(got.evicted_by) == evby


@pytest.mark.parametrize("seed", range(4))
def test_no_ports_is_the_plain_restatement(seed):
    snap, bound, cols, _ = random_case(seed)
    (entries, used), want = cols
    empty = ((entries, np.zeros_like(used)), np.zeros_like(want))
    none = np.zeros(bound.n, np.uint64)
    got, plain = R.preempt(snap, bound, empty, none), preempt_pdb_ref.preempt(snap, bound)
    assert _as_list(got) == _as_list(plain)
    for gang in (False, True):
        pods = W.queue(snap, gang=gang)
        got, plain = R.walk(snap, bound, empty, none, pods, gang), preempt_walk_ref.walk(snap, bound, pods, gang)
        assert _as_list(got, True) == _as_list(plain, True)
        np.testing.assert_array_equal(got.evicted_by, plain.evicted_by)


def test_random_cases_exercise_the_filter():
    """The random tables are not vacuous: the filter changes the answers of several preemptors across them."""
    changed = 0
    for seed in range(6):
        snap, bound, cols, ports = random_case(seed)
        got, plain = R.preempt(snap, bound, cols, ports), preempt_pdb_ref.preempt(snap, bound)
        changed += sum(a != b for a, b in zip(_as_list(got), _as_list(plain)))
    assert changed >= 5
