"""A SECOND, independent restatement of the reference's hot path — pure Python over Go-like objects
(dict-based ScalarResources, explicit loops), written from pkg/scheduler/core/core.go without looking
at oracle/bs_oracle.c.  Used only to cross-check the C oracle on small cases (tests/test_oracle_crosscheck.py):
two independent restatements agreeing is the strongest pin available while the Go reference cannot run.

Go semantics reproduced explicitly: int == int64 (Python ints are masked where Go would wrap),
uint32 arithmetic wraps, float32 via numpy.float32, float->int truncates.
"""
import numpy as np

M64 = (1 << 64) - 1
M32 = (1 << 32) - 1


def i64(x):
    x &= M64
    return x - (1 << 64) if x >> 63 else x


class Resource:  # nodeinfo.Resource
    def __init__(self):
        self.MilliCPU = 0
        self.Memory = 0
        self.EphemeralStorage = 0
        self.AllowedPodNumber = 0
        self.ScalarResources = {}

    def Add(self, other):  # Resource.Add(other.ResourceList())
        self.MilliCPU = i64(self.MilliCPU + other.MilliCPU)
        self.Memory = i64(self.Memory + other.Memory)
        self.EphemeralStorage = i64(self.EphemeralStorage + other.EphemeralStorage)
        self.AllowedPodNumber = i64(self.AllowedPodNumber + other.AllowedPodNumber)
        for k, v in other.ScalarResources.items():
            self.ScalarResources[k] = i64(self.ScalarResources.get(k, 0) + v)


def scale(alloc, percent):  # int64(float32(alloc) * percent)
    return int(np.float32(alloc) * np.float32(percent))


class Node:
    def __init__(self, nt, i):
        L = nt.lanes
        self.flags = int(nt.flags[i])
        self.alloc = Resource()
        self.req = Resource()
        a, r = nt.alloc[:, i], nt.requested[:, i]
        self.alloc.MilliCPU, self.alloc.Memory, self.alloc.EphemeralStorage, self.alloc.AllowedPodNumber = (int(x) for x in a[:4])
        self.req.MilliCPU, self.req.Memory, self.req.EphemeralStorage, self.req.AllowedPodNumber = (int(x) for x in r[:4])
        for d in range(4, L):
            if (int(nt.alloc_present[i]) >> d) & 1:
                self.alloc.ScalarResources[d] = int(a[d])
            if (int(nt.req_present[i]) >> d) & 1:
                self.req.ScalarResources[d] = int(r[d])
        self.n_pods = int(nt.pod_count[i])
        self.labels = int(nt.label_mask[i])
        self.taints = int(nt.taint_mask[i])


def check_fit(sel, tol, node):  # core.go:741-759
    return (node.labels & sel) == sel and (node.taints & ~tol & M64) == 0


def single_node_resource(node, sel, tol, percent):  # core.go:634-670
    left = Resource()
    if node.flags & 0x08:  # Taints() error
        return left
    if not check_fit(sel, tol, node):
        return left
    pod_count = node.req.AllowedPodNumber
    if pod_count == 0:
        pod_count = node.n_pods
    left.AllowedPodNumber = i64(scale(node.alloc.AllowedPodNumber, percent) - pod_count)
    left.MilliCPU = i64(scale(node.alloc.MilliCPU, percent) - node.req.MilliCPU)
    left.Memory = i64(scale(node.alloc.Memory, percent) - node.req.Memory)
    left.EphemeralStorage = i64(scale(node.alloc.EphemeralStorage, percent) - node.req.EphemeralStorage)
    for k, a in node.alloc.ScalarResources.items():
        if k not in node.req.ScalarResources:
            continue
        left.ScalarResources[k] = i64(scale(a, percent) - node.req.ScalarResources[k])
    return left


def compare_resource_and_require(left, req):  # core.go:672-699
    if left.Memory < req.Memory:
        return False
    if left.MilliCPU < req.MilliCPU:
        return False
    if left.EphemeralStorage < req.EphemeralStorage:
        return False
    if left.AllowedPodNumber < req.AllowedPodNumber:
        return False
    for k, v1 in req.ScalarResources.items():
        if k not in left.ScalarResources:
            if v1 != 0:
                return False
            continue
        if v1 > left.ScalarResources[k]:
            return False
    return True


def compare_cluster(nodes, sel, tol, need, percent):  # core.go:595-632
    running = Resource()
    for node in nodes:
        if node.flags & 0x07:  # nil info / nil Node() / unschedulable
            continue
        running.Add(single_node_resource(node, sel, tol, percent))
        if compare_resource_and_require(running, need):
            return True
    return False


def resource_from(vals, present, lanes):
    r = Resource()
    r.MilliCPU, r.Memory, r.EphemeralStorage, r.AllowedPodNumber = (int(x) for x in vals[:4])
    for d in range(4, lanes):
        if (int(present) >> d) & 1:
            r.ScalarResources[d] = int(vals[d])
    return r


def find_max_pg(gt, flags=None):  # core.go:701-739, table order
    flags = gt.flags if flags is None else flags
    max_idx, max_fin = -1, 0
    for g in range(gt.n):
        if flags[g] & 0x01:
            continue
        if not (flags[g] & 0x02):
            continue
        mm, sc = int(gt.min_member[g]), int(gt.scheduled[g])
        if ((mm - sc) & M32) <= 0:
            fin = 0
        else:
            if mm == 0:
                raise ZeroDivisionError("findMaxPG")
            fin = ((((int(gt.matched[g]) + sc) & M32) * 1000) & M32) // mm
        if fin > max_fin:
            max_fin, max_idx = fin, g
        elif fin == max_fin:
            if max_idx < 0 or (int(gt.scheduled[max_idx]) >= int(gt.min_member[max_idx]) and sc == 0):
                max_fin, max_idx = fin, g
    return max_idx, max_fin


def pre_allocated(gt, g, matched, min_res, min_res_present, has_minres):  # core.go:774-793
    out = Resource()
    mm = int(gt.min_member[g])
    not_finished = mm - matched if matched != 0 else mm - int(gt.scheduled[g])
    for _ in range(max(0, not_finished)):
        if has_minres:
            out.Add(resource_from(min_res, min_res_present, gt.lanes))
    if out.AllowedPodNumber == 0:
        out.AllowedPodNumber = mm + 1
    return out


def compare_pods(pt, gt, a, b):  # core.go:368-411
    p1, p2 = int(pt.priority[a]), int(pt.priority[b])
    g1, g2 = int(pt.gid[a]), int(pt.gid[b])
    n1, n2 = g1 == -1, g2 == -1
    if p1 > p2:
        return True
    if p1 == p2:
        if n1 and n2:
            return int(pt.ts_ns[a]) < int(pt.ts_ns[b])
        if n1:
            return True
        if n2:
            return False
    miss1 = n1 or g1 == -2 or bool(pt.flags[a] & 0x08)
    miss2 = n2 or g2 == -2 or bool(pt.flags[b] & 0x08)
    if miss1 or miss2:
        return False
    c1, c2 = int(gt.creation_ns[g1]), int(gt.creation_ns[g2])
    r1, r2 = int(gt.name_rank[g1]), int(gt.name_rank[g2])
    if p1 == p2 and c1 < c2:
        return True
    if p1 == p2 and c1 == c2 and r1 > r2:
        return True
    return p1 == p2 and c1 == c2 and r1 == r2 and int(pt.ts_ns[a]) < int(pt.ts_ns[b])


def prefilter_round(snap):
    """Round semantics of DESIGN.md §2 written straight from core.go:88-167 (+ :477-512)."""
    nt, pt, gt = snap.nodes, snap.pods, snap.groups
    L = nt.lanes
    nodes = [Node(nt, i) for i in range(nt.n)]
    flags = gt.flags.copy()
    rep_sel, rep_tol = gt.rep_sel.copy(), gt.rep_tol.copy()
    min_res, min_res_present = gt.min_res.copy(), gt.min_res_present.copy()
    for p in range(pt.n):  # fillOccupiedObj first-pod capture
        g = int(pt.gid[p])
        if g < 0 or g >= gt.n or (pt.flags[p] & 0x01) or (gt.flags[g] & 0x08):
            continue
        if not (flags[g] & 0x02):
            flags[g] |= 0x02
            rep_sel[g], rep_tol[g] = pt.sel_mask[p], pt.tol_mask[p]
        if not (flags[g] & 0x04):
            flags[g] |= 0x04
            for d in range(L):
                pres = d < 4 or ((int(pt.req_present[p]) >> d) & 1)
                min_res[d, g] = pt.req[d, p] if pres else 0
            min_res_present[g] = int(pt.req_present[p]) & ~0xF
    m, _ = find_max_pg(gt, flags)
    codes, denied = np.zeros(pt.n, np.uint8), np.zeros(gt.n, np.uint8)
    for p in range(pt.n):
        g = int(pt.gid[p])
        f = int(pt.flags[p])
        if g == -1 or (f & 0x01):
            continue
        if g < 0 or g >= gt.n:
            codes[p] = 1
            continue
        if gt.flags[g] & 0x08:
            codes[p] = 2
            continue
        if f & 0x02:
            codes[p] = 3
            continue
        if f & 0x04:
            codes[p] = 4
            continue
        if m < 0:
            continue
        matched = int(gt.matched[m])
        if matched == 0:
            need = pre_allocated(gt, g, 0, min_res[:, g], min_res_present[g], bool(flags[g] & 0x04))
            if not compare_cluster(nodes, int(rep_sel[g]), int(rep_tol[g]), need, 1.0):
                codes[p], denied[g] = 5, 1
            continue
        if m == g:
            continue
        need = pre_allocated(gt, m, matched, min_res[:, m], min_res_present[m], bool(flags[m] & 0x04))
        need.Add(resource_from(pt.req[:, p], int(pt.req_present[p]) & ~0xF, L))
        if not compare_cluster(nodes, int(rep_sel[m]), int(rep_tol[m]), need, 0.7):
            codes[p], denied[g] = 5, 1
    return codes, denied, m


def queue_order(pt, gt):
    """The queue order by Compare's key (core.go:379-408), ties in table order, and each pod's dense rank: the number
    of key changes before it along the order.  Lister misses sort after the resolvable groups."""
    P, G = pt.n, gt.n

    def key(p):
        g = int(pt.gid[p])
        if g == -1:
            return (-int(pt.priority[p]), 0, 0, 0, int(pt.ts_ns[p]))
        miss = g < 0 or g >= G or bool(pt.flags[p] & 0x08)
        creation = (1 << 63) - 1 if miss else int(gt.creation_ns[g])
        name = 0 if miss else -int(gt.name_rank[g])
        return (-int(pt.priority[p]), 1, creation, name, int(pt.ts_ns[p]))

    order = np.array(sorted(range(P), key=key), np.uint32)   # sorted() is stable
    rank = np.zeros(P, np.uint32)
    r = 0
    for i in range(P):
        if i and key(int(order[i])) != key(int(order[i - 1])):
            r += 1
        rank[order[i]] = r
    return order, rank


def round_outputs(snap):
    """The rest of a snapshot round (DESIGN.md §2) from the Go-like objects: fit matrix (the composite
    of core_test.go:108-110 behind the node guards and checkFit), builder-defined score, per-pod
    reductions, Permit verdict per group (core.go:303, uint32), and the queue order by Compare's key.
    Returns a dict of arrays shaped like the oracle's."""
    import functools
    nt, pt, gt = snap.nodes, snap.pods, snap.groups
    L, P, N, G = nt.lanes, pt.n, nt.n, gt.n
    nodes = [Node(nt, i) for i in range(N)]
    INT64_MIN = -(1 << 63)
    fit = np.zeros((P, N), bool)
    score = np.full((P, N), INT64_MIN, np.int64)
    for p in range(P):
        sel, tol = int(pt.sel_mask[p]), int(pt.tol_mask[p])
        req = resource_from(pt.req[:, p], int(pt.req_present[p]) & ~0xF, L)
        for i, node in enumerate(nodes):
            if (node.flags & 0x0F) or not check_fit(sel, tol, node):
                continue
            left = single_node_resource(node, sel, tol, 1.0)
            if not compare_resource_and_require(left, req):
                continue
            fit[p, i] = True
            diffs = [left.MilliCPU - req.MilliCPU, left.Memory - req.Memory,
                     left.EphemeralStorage - req.EphemeralStorage, left.AllowedPodNumber - req.AllowedPodNumber]
            diffs += [left.ScalarResources[k] - v for k, v in req.ScalarResources.items() if k in left.ScalarResources]
            score[p, i] = i64(min(diffs))
    feasible = fit.sum(axis=1).astype(np.uint32)
    best_node = np.full(P, -1, np.int32)
    best_score = np.full(P, INT64_MIN, np.int64)
    for p in range(P):
        if feasible[p]:
            best_node[p] = int(np.argmax(score[p]))   # first maximum = lowest index on ties
            best_score[p] = score[p, best_node[p]]
    codes, _, _ = prefilter_round(snap)
    contrib, in_round = np.zeros(G, np.int64), np.zeros(G, np.int64)
    for p in range(P):
        g = int(pt.gid[p])
        if 0 <= g < G:
            in_round[g] += 1
            if codes[p] == 0 and feasible[p]:
                contrib[g] += 1
    admit = np.zeros(G, np.uint8)
    for g in range(G):
        cnt = (int(gt.matched[g]) + int(contrib[g])) & M32
        if in_round[g] > 0 and contrib[g] == 0:
            admit[g] = 2
        else:
            admit[g] = 0 if cnt >= ((int(gt.min_member[g]) - int(gt.scheduled[g])) & M32) else 1

    order, rank = queue_order(pt, gt)
    return dict(fit=fit, score=score, feasible_count=feasible, best_node=best_node, best_score=best_score,
                admit=admit, order=order, rank=rank)


def get_left_resource(node):  # core.go:436-475
    """None when the reference returns nil (info == nil).  The scalar loop at :465-472 ranges over the
    Clone of a zero Resource, whose map is nil: it never runs, so no scalar key is ever reported."""
    if node.flags & 0x01:
        return None
    left = Resource()
    pod_count = node.req.AllowedPodNumber
    if pod_count == 0:
        pod_count = node.n_pods
    left.MilliCPU = i64(node.alloc.MilliCPU - node.req.MilliCPU)
    left.AllowedPodNumber = i64(node.alloc.AllowedPodNumber - pod_count)
    left.Memory = i64(node.alloc.Memory - node.req.Memory)
    left.EphemeralStorage = i64(node.alloc.EphemeralStorage - node.req.EphemeralStorage)
    return left


def filter_round(snap):
    """Filter / computeResourceSatisfied (core.go:170-191, :514-564) for every (pod, node) of a round,
    against the round's max group and its MinResources after the first-pod capture.
    Returns (passes[P][N] bool, code[P]) with code 0 pass-able, 1 group not found, 4 maxPGStatus nil."""
    nt, pt, gt = snap.nodes, snap.pods, snap.groups
    L = nt.lanes
    nodes = [Node(nt, i) for i in range(nt.n)]
    flags = gt.flags.copy()
    min_res, min_res_present = gt.min_res.copy(), gt.min_res_present.copy()
    for p in range(pt.n):  # fillOccupiedObj first-pod capture (as in prefilter_round)
        g = int(pt.gid[p])
        if g < 0 or g >= gt.n or (pt.flags[p] & 0x01) or (gt.flags[g] & 0x08):
            continue
        flags[g] |= 0x02
        if not (flags[g] & 0x04):
            flags[g] |= 0x04
            for d in range(L):
                pres = d < 4 or ((int(pt.req_present[p]) >> d) & 1)
                min_res[d, g] = pt.req[d, p] if pres else 0
            min_res_present[g] = int(pt.req_present[p]) & ~0xF
    m, _ = find_max_pg(gt, flags)
    max_single = None
    if m >= 0 and (flags[m] & 0x04):  # :525-528 maxSingleRequired = Resource{}.Add(*MinResources)
        max_single = Resource()
        max_single.Add(resource_from(min_res[:, m], int(min_res_present[m]), L))
    passes = np.zeros((pt.n, nt.n), bool)
    codes = np.zeros(pt.n, np.uint8)
    for p in range(pt.n):
        g = int(pt.gid[p])
        if g == -1:  # :171-174
            passes[p, :] = True
            continue
        if g < 0 or g >= gt.n:  # :177-180
            codes[p] = 1
            continue
        if m < 0:  # :525 dereferences sop.maxPGStatus == nil
            codes[p] = 4
            continue
        if m == g or max_single is None:  # :531-535 case 1; :542-544
            passes[p, :] = True
            continue
        for i, node in enumerate(nodes):
            left = get_left_resource(node)
            if left is None:  # :545-548
                continue
            cur = resource_from(pt.req[:, p], int(pt.req_present[p]) & ~0xF, L)
            cur.Add(max_single)  # :551-552
            if compare_resource_and_require(left, cur):  # case 2
                passes[p, i] = True
            elif not compare_resource_and_require(left, max_single):  # case 3
                passes[p, i] = True
    return passes, codes


def replay(snap, queue=None):
    """The reference's cycle, pod after pod, with mutable Go-like objects (DESIGN.md §10): PreFilter
    against the live state (core.go:88-167, fillOccupiedObj :477-512, AddToDenyCache :423-425), the
    pod assumed onto the first node in list order where A5 holds (NodeInfo.AddPod), Permit
    (core.go:268-309).  Written from core.go, independently of oracle/bs_oracle.c's bso_replay.
    Returns (prefilter[], node[], ready[]) per queue position."""
    nt, pt, gt = snap.nodes, snap.pods, snap.groups
    L = nt.lanes
    nodes = [Node(nt, i) for i in range(nt.n)]
    flags = [int(f) for f in gt.flags]
    matched = [int(m) for m in gt.matched]
    rep = [(int(s), int(t)) for s, t in zip(gt.rep_sel, gt.rep_tol)]
    min_res = [resource_from(gt.min_res[:, g], int(gt.min_res_present[g]), L) for g in range(gt.n)]

    class Live:  # what find_max_pg / pre_allocated read, seen through the mutable lists
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
            sel, tol = int(pt.sel_mask[p]), int(pt.tol_mask[p])
            for i, node in enumerate(nodes):
                if (node.flags & 0x0F) or not check_fit(sel, tol, node):
                    continue
                if compare_resource_and_require(single_node_resource(node, sel, tol, 1.0), req):
                    chosen = i
                    break
            if chosen >= 0:
                node = nodes[chosen]  # NodeInfo.AddPod: requested += request, the pod list grows
                node.req.MilliCPU = i64(node.req.MilliCPU + req.MilliCPU)
                node.req.Memory = i64(node.req.Memory + req.Memory)
                node.req.EphemeralStorage = i64(node.req.EphemeralStorage + req.EphemeralStorage)
                for k, v in req.ScalarResources.items():
                    node.req.ScalarResources[k] = i64(node.req.ScalarResources.get(k, int(nt.requested[k, chosen])) + v)
                node.n_pods += 1
                if g < 0 or g >= gt.n:
                    ready = 1
                else:
                    matched[g] += 1
                    if (matched[g] & M32) >= ((int(gt.min_member[g]) - int(gt.scheduled[g])) & M32):
                        flags[g] |= 0x01
                        ready = 1
        out_node.append(chosen)
        out_ready.append(ready)
    return np.array(out_pf, np.uint8), np.array(out_node, np.int32), np.array(out_ready, np.uint8)
