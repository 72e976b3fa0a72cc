"""A second, independent restatement of bs_replay_priority (include/bsched.h) in pure Python over the Go-like objects
of tests/pyref.py: tests/pyref.py's pod-at-a-time walk with the node choice as a hook, and a chooser built on
tests/pyref_priority.py's scorer.  Snapshots without affinity classes only, as tests/pyref.py's walk.  Used to
cross-check tests/replay_priority_ref.c on small cases."""
import numpy as np

from pyref import M32, Node, Resource, check_fit, compare_cluster, compare_resource_and_require, find_max_pg, i64, \
    resource_from, single_node_resource
from pyref_priority import score


def first_fit(nodes, pt, p, req):
    """tests/pyref.py's node choice: the first node in list order where the pod fits."""
    sel, tol = int(pt.sel_mask[p]), int(pt.tol_mask[p])
    for i, node in enumerate(nodes):
        if (node.flags & 0x0F) or not check_fit(sel, tol, node):
            continue
        if compare_resource_and_require(single_node_resource(node, sel, tol, 1.0), req):
            return i
    return -1


class PriorityChooser:
    """The best fitting node under the resource priorities on a live copy of the node non-zero column; ties to the
    lower index.  `assumed` grows the column (NodeInfo.AddPod)."""

    def __init__(self, node_nz, pod_nz, weights):
        self.node_nz = [[int(x) for x in row] for row in node_nz]
        self.pod_nz = pod_nz
        self.weights = weights

    def __call__(self, nodes, pt, p, req):
        sel, tol = int(pt.sel_mask[p]), int(pt.tol_mask[p])
        best, best_s = -1, None
        for i, node in enumerate(nodes):
            if (node.flags & 0x0F) or not check_fit(sel, tol, node):
                continue
            if not compare_resource_and_require(single_node_resource(node, sel, tol, 1.0), req):
                continue
            s = score(self.node_nz[0][i] + int(self.pod_nz[0][p]), node.alloc.MilliCPU,
                      self.node_nz[1][i] + int(self.pod_nz[1][p]), node.alloc.Memory, self.weights)
            if best < 0 or s > best_s:
                best, best_s = i, s
        return best

    def assumed(self, p, i):
        self.node_nz[0][i] += int(self.pod_nz[0][p])
        self.node_nz[1][i] += int(self.pod_nz[1][p])


def replay(snap, queue=None, choose=first_fit):
    """tests/pyref.py's replay with the node choice `choose(nodes, pods, p, request) -> index or -1`; a chooser with an
    `assumed(p, i)` method is told where each pod was assumed.  Returns (prefilter[], node[], ready[], after) with
    `after` the mutated node and group columns under bs_replay_result's names."""
    nt, pt, gt = snap.nodes, snap.pods, snap.groups
    L = nt.lanes
    nodes = [Node(nt, i) for i in range(nt.n)]
    flags = [int(f) for f in gt.flags]
    matched = [int(m) for m in gt.matched]
    rep = [(int(s), int(t)) for s, t in zip(gt.rep_sel, gt.rep_tol)]
    min_res = [resource_from(gt.min_res[:, g], int(gt.min_res_present[g]), L) for g in range(gt.n)]
    min_res_cols, min_res_present = gt.min_res.copy(), gt.min_res_present.copy()

    class Live:  # what find_max_pg reads, seen through the mutable lists
        n, lanes = gt.n, L
        min_member, scheduled = gt.min_member, gt.scheduled
    Live.matched = matched

    def need_of(g, matched_arg):
        out = Resource()
        mm = int(gt.min_member[g])
        not_finished = mm - matched_arg if matched_arg != 0 else mm - int(gt.scheduled[g])
        for _ in range(max(0, not_finished)):
            if flags[g] & 0x04:
                out.Add(min_res[g])
        if out.AllowedPodNumber == 0:
            out.AllowedPodNumber = mm + 1
        return out

    q = range(pt.n) if queue is None else [int(x) for x in queue]
    out_pf, out_node, out_ready = [], [], []
    for p in q:
        g, f = int(pt.gid[p]), int(pt.flags[p])
        req = resource_from(pt.req[:, p], int(pt.req_present[p]) & ~0xF, L)
        code = 0
        while True:  # PreFilter
            if g == -1 or (f & 0x01):
                break
            if g < 0 or g >= gt.n:
                code = 1
                break
            if flags[g] & 0x08:
                code = 2
                break
            if not (flags[g] & 0x02):
                flags[g] |= 0x02
                rep[g] = (int(pt.sel_mask[p]), int(pt.tol_mask[p]))
            if not (flags[g] & 0x04):
                flags[g] |= 0x04
                mr = Resource()
                mr.Add(req)
                min_res[g] = mr
                pres = int(pt.req_present[p])
                for d in range(L):
                    min_res_cols[d, g] = pt.req[d, p] if d < 4 or (pres >> d) & 1 else 0
                min_res_present[g] = pres & ~0xF
            if f & 0x02:
                code = 3
                break
            if f & 0x04:
                code = 4
                break
            m, _ = find_max_pg(Live, flags)
            if m < 0:
                break
            if matched[m] == 0:
                if not compare_cluster(nodes, rep[g][0], rep[g][1], need_of(g, 0), 1.0):
                    flags[g] |= 0x08
                    code = 5
                break
            if m == g:
                break
            need = need_of(m, matched[m])
            need.Add(req)
            if not compare_cluster(nodes, rep[m][0], rep[m][1], need, 0.7):
                flags[g] |= 0x08
                code = 5
            break
        out_pf.append(code)
        chosen, ready = -1, 0
        if code == 0:
            chosen = choose(nodes, pt, p, req)
            if chosen >= 0:
                node = nodes[chosen]  # NodeInfo.AddPod: requested += request, the pod list grows
                node.req.MilliCPU = i64(node.req.MilliCPU + req.MilliCPU)
                node.req.Memory = i64(node.req.Memory + req.Memory)
                node.req.EphemeralStorage = i64(node.req.EphemeralStorage + req.EphemeralStorage)
                for k, v in req.ScalarResources.items():
                    node.req.ScalarResources[k] = i64(node.req.ScalarResources.get(k, int(nt.requested[k, chosen])) + v)
                node.n_pods += 1
                if hasattr(choose, "assumed"):
                    choose.assumed(p, chosen)
                if g < 0 or g >= gt.n:
                    ready = 1
                else:
                    matched[g] += 1
                    if (matched[g] & M32) >= ((int(gt.min_member[g]) - int(gt.scheduled[g])) & M32):
                        flags[g] |= 0x01
                        ready = 1
        out_node.append(chosen)
        out_ready.append(ready)
    requested = nt.requested.copy()
    req_present = nt.req_present.copy()
    for i, node in enumerate(nodes):
        requested[:3, i] = (node.req.MilliCPU, node.req.Memory, node.req.EphemeralStorage)
        for k, v in node.req.ScalarResources.items():
            requested[k, i] = v
            req_present[i] |= np.uint32(1 << k)
    after = dict(node_requested=requested, node_pod_count=np.array([n.n_pods for n in nodes], np.int32),
                 node_req_present=req_present, group_matched=np.array(matched, np.uint32).reshape(gt.n),
                 group_flags=np.array(flags, np.uint8).reshape(gt.n), group_min_res=min_res_cols,
                 group_min_res_present=min_res_present,
                 group_rep_sel=np.array([r[0] for r in rep], np.uint64).reshape(gt.n),
                 group_rep_tol=np.array([r[1] for r in rep], np.uint64).reshape(gt.n))
    if hasattr(choose, "node_nz"):
        after["node_nonzero"] = np.array(choose.node_nz, np.int64).reshape(2, nt.n)
    return np.array(out_pf, np.uint8), np.array(out_node, np.int32), np.array(out_ready, np.uint8), after
