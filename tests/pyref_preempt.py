"""A second, independent restatement of bs_remove_pod and bs_preempt in pure Python over the Go-like objects of
tests/pyref.py (dict-based ScalarResources, explicit Go integer semantics, a real sort with MoreImportantPod), written
from core.go:203-260 and upstream's selectVictimsOnNode / pickOneNodeForPreemption [upstream, from memory] without
looking at the C restatement.  Used to cross-check tests/preempt_ref.c on small cases."""
import copy
import functools

from pyref import Node, check_fit, compare_resource_and_require, i64, resource_from, single_node_resource

GID_NONE, GID_MISSING = -1, -2
ALLOW, OFFLINE_ONLINE, NOT_FOUND, LOCKED, SAME_GROUP = range(5)


def remove_pod(gid_p, gid_v, locked_v):  # core.PreemptRemovePod
    pg_remove, offline_remove = gid_v, gid_v != GID_NONE
    pg_schedule, offline_schedule = gid_p, gid_p != GID_NONE
    if not offline_schedule and not offline_remove:
        return ALLOW
    if offline_schedule and not offline_remove:
        return OFFLINE_ONLINE

    def check_preemption():
        if pg_remove == GID_MISSING:          # podGroupStatusCache.Get == nil
            return "", NOT_FOUND
        if locked_v:                          # Status.Phase Scheduled / Running
            return "", LOCKED
        return ("g", pg_remove), None

    full_remove, err = check_preemption()
    if not offline_schedule and offline_remove:
        return ALLOW if err is None else err
    full_schedule = ("g", pg_schedule) if pg_schedule >= 0 else ("missing", pg_schedule)
    if full_remove == full_schedule:
        return SAME_GROUP
    return ALLOW if err is None else err


def _pod_fits(node, p_sel, p_tol, req):
    left = single_node_resource(node, p_sel, p_tol, 1.0)
    return compare_resource_and_require(left, req)


def _remove(node, vreq):  # NodeInfo.RemovePod on the copy
    node.req.MilliCPU = i64(node.req.MilliCPU - vreq.MilliCPU)
    node.req.Memory = i64(node.req.Memory - vreq.Memory)
    node.req.EphemeralStorage = i64(node.req.EphemeralStorage - vreq.EphemeralStorage)
    for k, v in vreq.ScalarResources.items():
        node.req.ScalarResources[k] = i64(node.req.ScalarResources[k] - v)
    node.n_pods -= 1


def _add(node, vreq):
    node.req.MilliCPU = i64(node.req.MilliCPU + vreq.MilliCPU)
    node.req.Memory = i64(node.req.Memory + vreq.Memory)
    node.req.EphemeralStorage = i64(node.req.EphemeralStorage + vreq.EphemeralStorage)
    for k, v in vreq.ScalarResources.items():
        node.req.ScalarResources[k] = i64(node.req.ScalarResources.get(k, 0) + v)
    node.n_pods += 1


def preempt(snap, bound, pods=None):
    """[(node or -1, [victim bound indices], n_candidates)] per pod."""
    nt, pt = snap.nodes, snap.pods
    L = nt.lanes
    aff_bits = getattr(snap, "aff_bits", None)
    aff_class = getattr(pt, "aff_class", None)
    nodes = [Node(nt, i) for i in range(nt.n)]
    on_node = [[] for _ in range(nt.n)]
    for v in range(bound.n):
        on_node[int(bound.node[v])].append(v)
    vreqs = []
    for v in range(bound.n):
        r = resource_from(bound.req[:, v], int(bound.req_present[v]), L)
        r.AllowedPodNumber = 0
        vreqs.append(r)

    def more_important(a, b):  # MoreImportantPod; the bound-table index decides the rest
        ka = (-int(bound.priority[a]), int(bound.start_ns[a]), a)
        kb = (-int(bound.priority[b]), int(bound.start_ns[b]), b)
        return -1 if ka < kb else (1 if ka > kb else 0)

    out = []
    for p in (range(pt.n) if pods is None else pods):
        p = int(p)
        sel, tol = int(pt.sel_mask[p]), int(pt.tol_mask[p])
        aff = 0xFFFFFFFF if aff_class is None else int(aff_class[p])
        req = resource_from(pt.req[:, p], int(pt.req_present[p]), L)
        prio = int(pt.priority[p])
        cands = []   # (node, victims) in node order
        for i, node in enumerate(nodes):
            if node.flags & 0x0F or not check_fit(sel, tol, node):
                continue
            if aff != 0xFFFFFFFF and not (int(aff_bits[aff, i // 32]) >> (i % 32)) & 1:
                continue
            left_keys = set(node.alloc.ScalarResources) & set(node.req.ScalarResources)
            if any(v != 0 and k not in left_keys for k, v in req.ScalarResources.items()):
                continue
            potential = [v for v in on_node[i] if int(bound.priority[v]) < prio]
            if any(remove_pod(int(pt.gid[p]), int(bound.gid[v]), int(bound.flags[v]) & 1) != ALLOW for v in potential):
                continue
            c = copy.deepcopy(node)
            for v in potential:
                _remove(c, vreqs[v])
            if not _pod_fits(c, sel, tol, req):
                continue
            victims = []
            for v in sorted(potential, key=functools.cmp_to_key(more_important)):
                _add(c, vreqs[v])
                if not _pod_fits(c, sel, tol, req):
                    _remove(c, vreqs[v])
                    victims.append(v)
            cands.append((i, victims))
        out.append((_pick(cands, bound), len(cands)))
    return [(n, v, c) for (n, v), c in out]


def _pick(cands, bound):  # pickOneNodeForPreemption, candidates in node order
    if not cands:
        return -1, []
    for i, vs in cands:
        if not vs:
            return i, vs
    prio = lambda v: int(bound.priority[v])
    m = min(prio(vs[0]) for _, vs in cands)
    s1 = [(i, vs) for i, vs in cands if prio(vs[0]) == m]
    sums = [sum(prio(v) + (1 << 31) for v in vs) for _, vs in s1]
    s2 = [c for c, s in zip(s1, sums) if s == min(sums)]
    n_min = min(len(vs) for _, vs in s2)
    s3 = [c for c in s2 if len(c[1]) == n_min]
    best, latest = s3[0], None
    for i, vs in s3:
        hp = prio(vs[0])
        earliest = min(int(bound.start_ns[v]) for v in vs if prio(v) == hp)
        if latest is None or earliest > latest:
            best, latest = (i, vs), earliest
    return best
