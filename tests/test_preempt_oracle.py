"""CPU: preemption (include/bsched.h bs_remove_pod / bs_preempt) on two CPU restatements — tests/preempt_ref.c, which
mutates a copy of each node and calls the C oracle's fit predicate, and tests/pyref_preempt.py — plus the RemovePod
messages of bs_format_remove_message and the seeded bound-pod generator.  The GPU is compared with the C restatement in
tests/test_gpu_preempt.py."""
import importlib
import itertools

import numpy as np
import pytest

import preempt_cases
import preempt_ref
import pyref_preempt
import randsnap

S = importlib.import_module("batch-scheduler_b200.snapshot")
E = importlib.import_module("batch-scheduler_b200.engine")

ONLINE, MISSING = S.GID_NONE, S.GID_MISSING
# (preemptor gid, victim gid, victim locked) -> verdict, the table of core.go:203-260 cell by cell
REMOVE_TABLE = [
    (ONLINE, ONLINE, 0, preempt_ref.ALLOW),
    (MISSING, ONLINE, 0, preempt_ref.OFFLINE_ONLINE),
    (0, ONLINE, 0, preempt_ref.OFFLINE_ONLINE),
    (ONLINE, MISSING, 0, preempt_ref.NOT_FOUND),
    (0, MISSING, 0, preempt_ref.NOT_FOUND),
    (MISSING, MISSING, 0, preempt_ref.NOT_FOUND),
    (ONLINE, 1, 1, preempt_ref.LOCKED),
    (0, 1, 1, preempt_ref.LOCKED),
    (0, 0, 1, preempt_ref.LOCKED),          # own group, locked: the phase message, not the same-group one
    (MISSING, 1, 1, preempt_ref.LOCKED),
    (ONLINE, 1, 0, preempt_ref.ALLOW),
    (0, 0, 0, preempt_ref.SAME_GROUP),
    (0, 1, 0, preempt_ref.ALLOW),
    (MISSING, 1, 0, preempt_ref.ALLOW),
]
MESSAGES = {
    preempt_ref.ALLOW: "",
    preempt_ref.OFFLINE_ONLINE: "offline pods p-0 are forbidden to preempt online v-0",
    preempt_ref.NOT_FOUND: "can not found pod group: ns/pg-v",
    preempt_ref.LOCKED: "pod belongs to Scheduled or Running pod group can not be scheduled",
    preempt_ref.SAME_GROUP: "podToSchedule and podToRemove belong to same pod group, do not preempt",
}


@pytest.mark.parametrize("gp,gv,locked,want", REMOVE_TABLE)
def test_remove_pod_table(gp, gv, locked, want):
    assert preempt_ref.remove_pod(gp, gv, locked) == want
    assert pyref_preempt.remove_pod(gp, gv, locked) == want
    assert E.format_remove_message(want, "p-0", "v-0", "ns/pg-v") == MESSAGES[want]


def test_remove_message_buffer_too_small():
    with pytest.raises(Exception):
        E.format_remove_message(preempt_ref.LOCKED, buf_len=10)


def _check(snap, bound, pods, want=None):
    got = preempt_ref.preempt(snap, bound, pods)
    py = pyref_preempt.preempt(snap, bound, pods)
    for k in range(len(pods)):
        assert (int(got.node[k]), got.victims_of(k), int(got.n_candidates[k])) == py[k], k
        if want is not None:
            assert (int(got.node[k]), got.victims_of(k)) == tuple(want[k]), k
    return got


@pytest.mark.parametrize("name", sorted(preempt_cases.cases()))
def test_hand_built_case(name):
    snap, bound, pods, want = preempt_cases.cases()[name]
    _check(snap, bound, pods, want)


RAND = list(itertools.product(range(51), (4, 5, 9, 16)))


@pytest.mark.parametrize("seed,L", RAND)
def test_c_restatement_agrees_with_pyref_random(seed, L):
    snap = randsnap.random_snapshot(seed, P=8, N=12, G=4, L=L, aff=3 if seed % 2 else 0)
    bound = S.bound_pods(snap, seed, max_per_node=5, priorities=(-5, 0, 1, 100, 2**31 - 1, -2**31), n_starts=3,
                         online=0.3 if seed % 3 else 0.0, locked=0.2 if seed % 4 else 0.0)
    _check(snap, bound, np.arange(snap.pods.n))


def test_bound_pods_generator():
    snap = randsnap.random_snapshot(3, P=4, N=40, G=6, L=7)
    bt = S.bound_pods(snap, 1)
    nt = snap.nodes
    per_node = np.bincount(bt.node, minlength=nt.n)
    assert np.all(per_node <= np.clip(nt.pod_count, 0, None))
    assert np.all((bt.req_present & ~np.uint32(0xF) & ~nt.req_present[bt.node]) == 0)
    for d in range(3):   # lanes 0-2 split the node's requested amounts
        np.testing.assert_array_equal(np.bincount(bt.node, weights=bt.req[d], minlength=nt.n)[per_node > 0],
                                      nt.requested[d][per_node > 0])
    assert set(np.unique(bt.gid)) <= set(range(-2, snap.groups.n))
    assert np.all(bt.flags[bt.gid < 0] == 0)
    again = S.bound_pods(snap, 1)
    for f in bt.__dataclass_fields__:
        np.testing.assert_array_equal(getattr(bt, f), getattr(again, f))
