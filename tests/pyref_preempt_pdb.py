"""The pure-Python restatement of bs_preempt with PodDisruptionBudget-violating bound pods (include/bsched.h
BS_BOUND_PDB_VIOLATING), over the Go-like objects of tests/pyref.py, written from upstream's selectVictimsOnNode /
filterPodsWithPDBViolation / pickOneNodeForPreemption [upstream, from memory] without looking at the C restatement
tests/preempt_pdb_ref.c.  RemovePod and the node-copy arithmetic are tests/pyref_preempt.py's, which restates
preemption without budgets.  A bound row flagged PDB_VIOLATING is a pod filterPodsWithPDBViolation puts on the
violating side.  Used to cross-check tests/preempt_pdb_ref.c on small cases."""
import copy
import functools

from pyref import Node, check_fit, resource_from
from pyref_preempt import ALLOW, _add, _pod_fits, _remove, remove_pod

PDB_VIOLATING = 0x02


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
            potential.sort(key=functools.cmp_to_key(more_important))
            violating = [v for v in potential if int(bound.flags[v]) & PDB_VIOLATING]
            non_violating = [v for v in potential if not int(bound.flags[v]) & PDB_VIOLATING]
            victims, n_violating = [], 0
            for part, is_violating in ((violating, True), (non_violating, False)):
                for v in part:   # reprievePod
                    _add(c, vreqs[v])
                    if not _pod_fits(c, sel, tol, req):
                        _remove(c, vreqs[v])
                        victims.append(v)
                        n_violating += is_violating
            cands.append((i, victims, n_violating))
        out.append((_pick(cands, bound), len(cands)))
    return [(n, v, c) for (n, v), c in out]


def _pick(cands, bound):  # pickOneNodeForPreemption, candidates (node, victims, violating count) in node order
    if not cands:
        return -1, []
    for i, vs, _ in cands:
        if not vs:
            return i, vs
    fewest = min(nvio for _, _, nvio in cands)
    s0 = [(i, vs) for i, vs, nvio in cands if nvio == fewest]
    prio = lambda v: int(bound.priority[v])
    m = min(prio(vs[0]) for _, vs in s0)   # upstream takes victims[0] as the highest
    s1 = [(i, vs) for i, vs in s0 if prio(vs[0]) == m]
    sums = [sum(prio(v) + (1 << 31) for v in vs) for _, vs in s1]
    s2 = [c for c, s in zip(s1, sums) if s == min(sums)]
    n_min = min(len(vs) for _, vs in s2)
    s3 = [c for c in s2 if len(c[1]) == n_min]
    best, latest = s3[0], None
    for i, vs in s3:
        hp = max(prio(v) for v in vs)   # GetEarliestPodStartTime: the true maximum
        earliest = min(int(bound.start_ns[v]) for v in vs if prio(v) == hp)
        if latest is None or earliest > latest:
            best, latest = (i, vs), earliest
    return best
