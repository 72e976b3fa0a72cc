"""Hand-built preemption cases with PodDisruptionBudget-violating bound pods (include/bsched.h BS_BOUND_PDB_VIOLATING),
each forcing one decision the budgets change in selectVictimsOnNode or pickOneNodeForPreemption.  The preemptors have
priority 100 and are online unless a case says otherwise; the bound pods are online.  A case is (snapshot, bound-pod
table, preemptor pod indices, expected [(node, victims)], expected [(node, victims)] with every bit cleared).
Lanes as in tests/preempt_cases.py: 0 cpu, 1 memory, 2 ephemeral storage, 3 pods, 4 a scalar resource."""
import importlib

import numpy as np

import preempt_cases

S = importlib.import_module("batch-scheduler_b200.snapshot")


def _bound(rows):
    """rows: preempt_cases rows plus "vio" (the pod violates a PodDisruptionBudget)."""
    bt = preempt_cases._bound(rows)
    for v, r in enumerate(rows):
        if r.get("vio"):
            bt.flags[v] |= S.BOUND_PDB_VIOLATING
    return bt


def without_bits(bound):
    """The same table with every BS_BOUND_PDB_VIOLATING bit cleared."""
    bt = bound.copy()
    bt.flags &= np.uint8(~S.BOUND_PDB_VIOLATING & 0xFF)
    return bt


def cases():
    """name -> (snapshot, bound table, preemptors, expected, expected without the bits)."""
    c = {}
    # 1. the violating pod A is reprieved first and stays; B goes.  Without the bit B is reprieved first, A goes.
    c["reprieve_order"] = (
        preempt_cases._snap([{"cpu_alloc": 4000, "cpu_req": 4000}], [{"cpu": 2000}]),
        _bound([{"node": 0, "cpu": 2000, "prio": 10, "vio": True}, {"node": 0, "cpu": 2000, "prio": 20}]),
        [0], [(0, [1])], [(0, [0])])
    # 2. node 0 evicts one violating pod of priority 0, node 1 one non-violating pod of priority 50: fewest violations
    # wins over the lower priority
    c["fewest_violations"] = (
        preempt_cases._snap([{}, {}], [{"cpu": 10}]),
        _bound([{"node": 0, "cpu": 10, "prio": 0, "vio": True}, {"node": 1, "cpu": 10, "prio": 50}]),
        [0], [(1, [1])], [(0, [0])])
    # 3. one violation on each node; node 0's victims are [V (0), W (40)], so its "highest" priority is V's 0 (the
    # first victim's), below node 1's 10: node 0 wins, where a true-maximum rule would pick node 1
    c["first_victim_quirk"] = (
        preempt_cases._snap([{"cpu_alloc": 2000, "cpu_req": 2000}, {"cpu_alloc": 2000, "cpu_req": 2000}],
                            [{"cpu": 2000}]),
        _bound([{"node": 0, "cpu": 1000, "prio": 0, "vio": True}, {"node": 0, "cpu": 1000, "prio": 40},
                {"node": 1, "cpu": 2000, "prio": 10, "vio": True}]),
        [0], [(0, [0, 1])], [(1, [2])])
    # 4. criteria 1-4 tie; the start criterion reads the earliest start among the priority-40 victims (node 0: 1,
    # node 1: 5), not the first victim's (node 0: 5, node 1: 1): node 1
    c["start_true_maximum"] = (
        preempt_cases._snap([{"cpu_alloc": 2000, "cpu_req": 2000}, {"cpu_alloc": 2000, "cpu_req": 2000}],
                            [{"cpu": 2000}]),
        _bound([{"node": 0, "cpu": 1000, "prio": 0, "start": 5, "vio": True},
                {"node": 0, "cpu": 1000, "prio": 40, "start": 1},
                {"node": 1, "cpu": 1000, "prio": 0, "start": 1, "vio": True},
                {"node": 1, "cpu": 1000, "prio": 40, "start": 5}]),
        [0], [(1, [2, 3])], [(1, [3, 2])])
    # 5. the bit on pods at or above the preemptor's priority changes nothing: they are never potential victims
    c["bit_above_preemptor"] = (
        preempt_cases._snap([{}, {}], [{"cpu": 5}]),
        _bound([{"node": 0, "cpu": 5, "prio": 100, "vio": True}, {"node": 0, "cpu": 5, "prio": 1},
                {"node": 1, "cpu": 5, "prio": 200, "vio": True}, {"node": 1, "cpu": 5, "prio": 2}]),
        [0], [(0, [1])], [(0, [1])])
    # 6. a violating pod that RemovePod refuses still drops its node: node 0's pod is in a locked group (it would win
    # for the online preemptor on the index), node 1's is online (refused for the offline preemptor of group 1)
    c["refused_violating"] = (
        preempt_cases._snap([{}, {}, {}], [{"cpu": 10}, {"cpu": 10, "gid": 1}], groups=3),
        _bound([{"node": 0, "cpu": 10, "prio": 1, "gid": 2, "locked": True, "vio": True},
                {"node": 1, "cpu": 10, "prio": 1, "vio": True},
                {"node": 2, "cpu": 10, "prio": 50, "gid": 0, "vio": True}]),
        [0, 1], [(1, [1]), (2, [2])], [(1, [1]), (2, [2])])
    return c
