"""Hand-built cases of the sequential preemption walk (include/bsched.h bs_preempt_walk), each with its answers
written out: what the walk gives and what bs_preempt gives the same preemptors as independent what-ifs.  A case is
(snapshot, bound-pod table, preemptor pod indices, gang, expected walk [(node, victims, outcome)], expected bs_preempt
[(node, victims)]).  Lanes as in tests/preempt_cases.py: 0 cpu, 1 memory, 2 ephemeral storage, 3 pods, 4 a scalar
resource."""
import importlib

import numpy as np

import pdb_cases
import preempt_cases
import randsnap

S = importlib.import_module("batch-scheduler_b200.snapshot")

NONE, NOMINATED, ROLLED_BACK = range(3)   # BS_WALK_*

# Two nodes of cpu 4000, fully requested by 2000-cpu bound pods of the unlocked group h = 0 (not online pods: RemovePod
# refuses to let a gang member evict an online pod).  Node 0 holds A (prio 0, start 50) and B (prio 0, start 100);
# node 1 holds D (prio 5) and C (prio 0, start 100).  Rows: A = 0, B = 1, D = 2, C = 3.
_TWO_NODES = [{"cpu_alloc": 4000, "cpu_req": 4000}, {"cpu_alloc": 4000, "cpu_req": 4000}]
_ABDC = [{"node": 0, "cpu": 2000, "prio": 0, "start": 50, "gid": 0},
         {"node": 0, "cpu": 2000, "prio": 0, "start": 100, "gid": 0},
         {"node": 1, "cpu": 2000, "prio": 5, "start": 0, "gid": 0},
         {"node": 1, "cpu": 2000, "prio": 0, "start": 100, "gid": 0}]


def cases():
    c = {}
    # Two online preemptors of prio 10, cpu 2000.  bs_preempt gives both node 0, [B].  In the walk the nominated p1
    # leaves only A on node 0, whose earlier start loses the start criterion to C's on node 1.
    c["nomination_moves_second"] = (
        preempt_cases._snap(_TWO_NODES, [{"cpu": 2000, "prio": 10}, {"cpu": 2000, "prio": 10}]),
        preempt_cases._bound(_ABDC), [0, 1], False,
        [(0, [1], NOMINATED), (1, [3], NOMINATED)], [(0, [1]), (0, [1])])
    # cpu 3000: a 3-pod gang of group g = 1, then an online pod q.  p1 takes node 0 ([A, B]: node 1's first victim D
    # has the higher priority), p2 node 1 ([D, C]), p3 finds nothing, so the unit rolls back and q sees the
    # uploaded state: node 0, [A, B].
    gang = [{"cpu": 3000, "prio": 10, "gid": 1}] * 3 + [{"cpu": 3000, "prio": 10}]
    c["gang_rolls_back"] = (
        preempt_cases._snap(_TWO_NODES, gang), preempt_cases._bound(_ABDC), [0, 1, 2, 3], True,
        [(-1, [], ROLLED_BACK)] * 3 + [(0, [0, 1], NOMINATED)], [(0, [0, 1])] * 4)
    # the same list without gang units: p1 and p2 keep their nodes and q finds none
    c["gang_off_keeps_members"] = (
        preempt_cases._snap(_TWO_NODES, gang), preempt_cases._bound(_ABDC), [0, 1, 2, 3], False,
        [(0, [0, 1], NOMINATED), (1, [2, 3], NOMINATED), (-1, [], NONE), (-1, [], NONE)], [(0, [0, 1])] * 4)
    # The pods lane counted by len(Pods()) (requested[3] == 0): two slots, both held by bound pods of prio 1 (row 0)
    # and 2 (row 1).  p1 evicts row 0; the nominated p1 holds a slot, so p2 must evict row 1; p3 finds two nominated
    # pods, which are never victims.
    c["pods_lane_by_count"] = (
        preempt_cases._snap([{"cpu_req": 0, "pods_alloc": 2, "pod_count": 2}], [{"pods": 1}] * 3),
        preempt_cases._bound([{"node": 0, "prio": 1}, {"node": 0, "prio": 2}]), [0, 1, 2], False,
        [(0, [0], NOMINATED), (0, [1], NOMINATED), (-1, [], NONE)], [(0, [0])] * 3)
    # PodDisruptionBudget-violating rows across steps: node 0 holds W (row 0), node 1 the violating V (row 1).  p1
    # takes node 0 (no violation); p2 then has only node 1 and evicts V.
    c["violating_row_next_step"] = (
        preempt_cases._snap([{}, {}], [{"cpu": 10}, {"cpu": 10}]),
        pdb_cases._bound([{"node": 0, "cpu": 10, "prio": 0}, {"node": 1, "cpu": 10, "prio": 0, "vio": True}]),
        [0, 1], False, [(0, [0], NOMINATED), (1, [1], NOMINATED)], [(0, [0]), (0, [0])])
    return c


def queue(snap, pods=None, gang=False):
    """A walk list of `pods` (all when None) in queue order: priority descending, then the group, then the index.
    With gang, every group's pods are first given one priority (the first pod's), so that each group is contiguous."""
    pt = snap.pods
    pods = np.arange(pt.n) if pods is None else np.asarray(pods)
    if gang:
        for g in np.unique(pt.gid[pods]):
            if g >= 0:
                members = pods[pt.gid[pods] == g]
                pt.priority[members] = pt.priority[members[0]]
    return sorted(pods.tolist(), key=lambda p: (-int(pt.priority[p]), int(pt.gid[p]), p))


def random_table(seed, L, violating, P=10, N=8, G=3, max_per_node=5):
    """A random table where preemptors compete: most nodes full, a few preemptor priorities, half the pods online."""
    snap = randsnap.random_snapshot(seed, P=P, N=N, G=G, L=L, aff=3 if seed % 2 else 0)
    rng = np.random.default_rng(seed + 1000)
    full = rng.random(N) < 0.7
    snap.nodes.requested[:3, full] = snap.nodes.alloc[:3, full]
    snap.pods.gid[rng.random(P) < 0.5] = S.GID_NONE
    snap.pods.priority[:] = rng.choice([2, 1000, 2**31 - 1], P)
    bound = S.bound_pods(snap, seed, max_per_node=max_per_node, priorities=(-5, 0, 1, 100, 2**31 - 1, -2**31),
                         n_starts=3, online=0.3 if seed % 3 else 0.0, locked=0.2 if seed % 4 else 0.0,
                         violating=violating)
    return snap, bound
