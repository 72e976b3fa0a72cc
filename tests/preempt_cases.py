"""Hand-built preemption cases (include/bsched.h bs_preempt), each forcing one decision of selectVictimsOnNode or
pickOneNodeForPreemption.  A case is (snapshot, bound-pod table, preemptor pod indices, expected [(node, victims)]).
Lanes: 0 cpu, 1 memory, 2 ephemeral storage, 3 pods, 4 a scalar resource (gpu)."""
import importlib

import numpy as np

S = importlib.import_module("batch-scheduler_b200.snapshot")

L = 5
GPU = 1 << 4


def _snap(nodes, pods, groups=2):
    """nodes: dicts (cpu_alloc, cpu_req, pod_count, pods_alloc, pods_req, gpu_alloc, gpu_req, flags, label, taint);
    pods: dicts (cpu, pods, gpu, prio, gid, sel, tol)."""
    N, P = len(nodes), len(pods)
    nt = S.NodeTable.empty(N, L)
    for i, nd in enumerate(nodes):
        nt.alloc[:, i] = [nd.get("cpu_alloc", 10), 1000, 1000, nd.get("pods_alloc", 100), nd.get("gpu_alloc", 0)]
        nt.requested[:, i] = [nd.get("cpu_req", 10), 0, 0, nd.get("pods_req", 0), nd.get("gpu_req", 0)]
        nt.pod_count[i] = nd.get("pod_count", 10)
        if "gpu_alloc" in nd:
            nt.alloc_present[i] = GPU
            nt.req_present[i] = GPU
        nt.flags[i] = nd.get("flags", 0)
        nt.label_mask[i] = nd.get("label", 0)
        nt.taint_mask[i] = nd.get("taint", 0)
    pt = S.PodTable.empty(P, L)
    for p, pd in enumerate(pods):
        pt.req[:, p] = [pd.get("cpu", 0), 0, 0, pd.get("pods", 0), pd.get("gpu", 0)]
        pt.req_present[p] = GPU if "gpu" in pd else 0
        pt.priority[p] = pd.get("prio", 100)
        pt.gid[p] = pd.get("gid", S.GID_NONE)
        pt.sel_mask[p] = pd.get("sel", 0)
        pt.tol_mask[p] = pd.get("tol", 0)
    gt = S.GroupTable.empty(groups, L)
    gt.min_member[:] = 1
    return S.Snapshot(nt, pt, gt, "preempt-case")


def _bound(rows):
    """rows: dicts (node, cpu, gpu, prio, start, gid, locked)."""
    bt = S.BoundPodTable.empty(len(rows), L)
    for v, r in enumerate(rows):
        bt.node[v] = r["node"]
        bt.req[:, v] = [r.get("cpu", 0), 0, 0, 0, r.get("gpu", 0)]
        bt.req_present[v] = GPU if "gpu" in r else 0
        bt.priority[v] = r.get("prio", 1)
        bt.start_ns[v] = r.get("start", 0)
        bt.gid[v] = r.get("gid", S.GID_NONE)
        bt.flags[v] = S.BOUND_GROUP_LOCKED if r.get("locked") else 0
    return bt


def cases():
    """name -> (snapshot, bound table, preemptors, expected [(node, victims)] per preemptor)."""
    c = {}
    # one refusable potential victim rules node 0 out although the pod would not need it evicted
    c["refusable_unneeded_victim"] = (
        _snap([{}, {}], [{"cpu": 5}]),
        _bound([{"node": 0, "cpu": 10}, {"node": 0, "cpu": 0, "gid": 0, "locked": True}, {"node": 1, "cpu": 10}]),
        [0], [(1, [2])])
    # equal priority is never a victim
    c["equal_priority_not_victim"] = (
        _snap([{}], [{"cpu": 5, "prio": 7}]), _bound([{"node": 0, "cpu": 10, "prio": 7}]), [0], [(-1, [])])
    # reprieve goes most important first: the high-priority pod stays, the low one goes
    c["reprieve_order"] = (
        _snap([{"cpu_req": 8}], [{"cpu": 6, "prio": 10}]),
        _bound([{"node": 0, "cpu": 4, "prio": 1}, {"node": 0, "cpu": 4, "prio": 5}]), [0], [(0, [0])])
    # equal priority: the earlier start is reprieved first; equal start: the lower index
    c["tie_start"] = (
        _snap([{"cpu_req": 8}], [{"cpu": 6}]),
        _bound([{"node": 0, "cpu": 4, "start": 2}, {"node": 0, "cpu": 4, "start": 1}]), [0], [(0, [0])])
    c["tie_index"] = (
        _snap([{"cpu_req": 8}], [{"cpu": 6}]),
        _bound([{"node": 0, "cpu": 4, "start": 1}, {"node": 0, "cpu": 4, "start": 1}]), [0], [(0, [1])])
    # the pick's criteria, each deciding alone (the winner is never the first candidate)
    c["pick_highest_priority"] = (
        _snap([{}, {}], [{"cpu": 10}]),
        _bound([{"node": 0, "cpu": 10, "prio": 5}, {"node": 1, "cpu": 10, "prio": 3}]), [0], [(1, [1])])
    c["pick_sum"] = (
        _snap([{}, {}], [{"cpu": 10}]),
        _bound([{"node": 0, "cpu": 5, "prio": 3}, {"node": 0, "cpu": 5, "prio": 2},
                {"node": 1, "cpu": 5, "prio": 3}, {"node": 1, "cpu": 5, "prio": 1}]), [0], [(1, [2, 3])])
    imin = -2 ** 31
    c["pick_count"] = (
        _snap([{}, {}], [{"cpu": 10, "prio": 0}]),
        _bound([{"node": 0, "cpu": 5, "prio": imin}, {"node": 0, "cpu": 5, "prio": imin},
                {"node": 1, "cpu": 10, "prio": imin}]), [0], [(1, [2])])
    c["pick_latest_start"] = (
        _snap([{}, {}], [{"cpu": 10}]),
        _bound([{"node": 0, "cpu": 10, "start": 5}, {"node": 1, "cpu": 10, "start": 9}]), [0], [(1, [1])])
    c["pick_index"] = (
        _snap([{}, {}], [{"cpu": 10}]),
        _bound([{"node": 0, "cpu": 10}, {"node": 1, "cpu": 10}]), [0], [(0, [0])])
    # a candidate without victims wins at once
    c["zero_victims"] = (
        _snap([{}, {"cpu_req": 0}], [{"cpu": 10}]),
        _bound([{"node": 0, "cpu": 10}, {"node": 1, "cpu": 0, "prio": 1000}]), [0], [(1, [])])
    # the pods lane: with requested[3] == 0 the pod count frees slots, otherwise removal does not help
    c["pods_lane_by_count"] = (
        _snap([{"cpu_req": 0, "pods_alloc": 2, "pod_count": 2}], [{"pods": 1}]),
        _bound([{"node": 0, "prio": 1}, {"node": 0, "prio": 2}]), [0], [(0, [0])])
    c["pods_lane_requested"] = (
        _snap([{"cpu_req": 0, "pods_alloc": 2, "pods_req": 2, "pod_count": 2}], [{"pods": 1}]),
        _bound([{"node": 0, "prio": 1}, {"node": 0, "prio": 2}]), [0], [(-1, [])])
    # scalar-keyed victims free the scalar lane
    c["scalar_victims"] = (
        _snap([{"cpu_req": 0, "gpu_alloc": 4, "gpu_req": 4}], [{"gpu": 2}]),
        _bound([{"node": 0, "gpu": 2, "prio": 1}, {"node": 0, "gpu": 2, "prio": 2}]), [0], [(0, [0])])
    # unschedulable, selector and taint failures cannot be resolved by preemption
    c["unresolvable_nodes"] = (
        _snap([{"flags": S.NODE_UNSCHEDULABLE}, {"label": 0}, {"label": 1, "taint": 2}, {"label": 1}],
              [{"cpu": 10, "sel": 1}]),
        _bound([{"node": k, "cpu": 10, "start": 9 - k} for k in range(4)]), [0], [(3, [3])])
    # an offline preemptor is kept off a node with a lower-priority online pod; an online one is not
    c["offline_vs_online"] = (
        _snap([{}, {}], [{"cpu": 5, "gid": 0}, {"cpu": 5}]),
        _bound([{"node": 0, "cpu": 10, "prio": 1}, {"node": 0, "cpu": 0, "prio": 1},
                {"node": 1, "cpu": 10, "prio": 5, "gid": 1}]), [0, 1], [(1, [2]), (0, [0])])
    # an offline preemptor does not evict pods of its own group; a locked group is never evicted
    c["same_group_and_locked"] = (
        _snap([{}, {}, {}], [{"cpu": 10, "gid": 0}]),
        _bound([{"node": 0, "cpu": 10, "gid": 0}, {"node": 1, "cpu": 10, "gid": 1, "locked": True},
                {"node": 2, "cpu": 10, "gid": 1, "prio": 50}]), [0], [(2, [2])])
    return c
