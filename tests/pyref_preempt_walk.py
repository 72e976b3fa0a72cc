"""The pure-Python restatement of bs_preempt_walk (include/bsched.h) over the Go-like objects of tests/pyref.py, written
without looking at the C restatement tests/preempt_walk_ref.c: kube-scheduler's one-pod-per-cycle preemption, where
each pod's victims are gone and the pod is nominated to its node before the next preemptor is considered.  One step is
tests/pyref_preempt_pdb.py's single-pod preemption on the live node table and the bound pods not yet evicted.  Used to
cross-check tests/preempt_walk_ref.c on small cases."""
import numpy as np

import pyref_preempt_pdb

NONE, NOMINATED, ROLLED_BACK = range(3)   # BS_WALK_*


def _units(snap, pods, gang):
    """The walk's units as lists of positions: with gang, a run of preemptors of one group of the table; else, and
    for a gid that names no group (negative or >= n_groups), one each."""
    units = []
    for i, p in enumerate(pods):
        g = int(snap.pods.gid[p])
        if gang and 0 <= g < snap.groups.n and units and int(snap.pods.gid[pods[units[-1][-1]]]) == g:
            units[-1].append(i)
        else:
            units.append([i])
    return units


def walk(snap, bound, pods, gang=False):
    """[(node or -1, [victim bound indices], n_candidates, outcome)] per preemptor, and evicted_by [V]."""
    pods = [int(p) for p in pods]
    live = snap.copy()   # the node table is the live state; the rest is read only
    nt, pt = live.nodes, live.pods
    evicted_by = [-1] * bound.n
    out = [None] * len(pods)
    for unit in _units(snap, pods, gang):
        saved = (nt.copy(), list(evicted_by))
        failed = False
        for i in unit:
            rows = [v for v in range(bound.n) if evicted_by[v] < 0]
            sub = _rows(bound, rows)
            (node, victims, cand), = pyref_preempt_pdb.preempt(live, sub, [pods[i]])
            victims = [rows[v] for v in victims]
            if node < 0:
                failed = True
                out[i] = (-1, [], cand, NONE)
                continue
            out[i] = (node, victims, cand, NOMINATED)
            p = pods[i]
            for v in victims:            # NodeInfo.RemovePod
                evicted_by[v] = i
                for d in range(nt.lanes):
                    if d != 3 and (d < 4 or (int(bound.req_present[v]) >> d) & 1):
                        nt.requested[d, node] -= bound.req[d, v]
                nt.pod_count[node] -= 1
            for d in range(nt.lanes):     # NodeInfo.AddPod of the nominated pod
                if d != 3 and (d < 4 or (int(pt.req_present[p]) >> d) & 1):
                    nt.requested[d, node] += pt.req[d, p]
                    if d >= 4:
                        nt.req_present[node] |= np.uint32(1 << d)
            nt.pod_count[node] += 1
        if gang and failed:
            live.nodes, evicted_by = saved
            nt = live.nodes
            for i in unit:
                out[i] = (-1, [], out[i][2], ROLLED_BACK)
    return out, evicted_by


def _rows(bound, rows):
    idx = np.asarray(rows, np.int64)
    return type(bound)(bound.node[idx], bound.req[:, idx], bound.req_present[idx], bound.gid[idx],
                       bound.priority[idx], bound.start_ns[idx], bound.flags[idx]) if len(rows) else \
        type(bound).empty(0, bound.lanes)
