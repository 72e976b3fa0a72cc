"""The pure-Python restatement of bs_preempt and bs_preempt_walk under the PodFitsHostPorts filter (include/bsched.h
bs_upload_bound_host_ports), over the Go-like objects of tests/pyref.py, written from upstream's selectVictimsOnNode /
podPassesFiltersOnNode / HostPortInfo [upstream, from memory] without looking at the C restatement
tests/preempt_host_ports_ref.c.  A node's used ports are a Python set of (ip, protocol, port) tuples: RemovePod
discards its pod's tuples whoever else holds them, and nominated pods join a copy of the set at filter time only.
RemovePod, the node-copy arithmetic and the pick are tests/pyref_preempt.py's and tests/pyref_preempt_pdb.py's.  Used
to cross-check tests/preempt_host_ports_ref.c on small cases."""
import copy
import functools

import numpy as np

from pyref import Node, check_fit, resource_from
from pyref_preempt import ALLOW, _add, _pod_fits, _remove, remove_pod
from pyref_preempt_pdb import PDB_VIOLATING, _pick
from pyref_preempt_walk import NOMINATED, NONE, ROLLED_BACK, _units

ANY = 0


def _tuples(entries, mask):
    return {tuple(int(x) for x in entries[k]) for k in range(len(entries)) if (int(mask) >> k) & 1}


def _conflict(used, want):   # HostPortInfo.CheckConflict over every wanted tuple
    return any(u[1] == w[1] and u[2] == w[2] and (w[0] == ANY or u[0] == ANY or u[0] == w[0])
               for w in want for u in used)


def _preempt_one(snap, bound, rows, entries, used, nom, ports, p):
    """(node or -1, [victims among `rows`], n_candidates) of pod p: rows are the live bound indices, used / nom each
    node's bound and nominated tuple sets."""
    nt, pt = snap.nodes, snap.pods
    L = nt.lanes
    aff_bits = getattr(snap, "aff_bits", None)
    aff_class = getattr(pt, "aff_class", None)
    sel, tol = int(pt.sel_mask[p]), int(pt.tol_mask[p])
    aff = 0xFFFFFFFF if aff_class is None else int(aff_class[p])
    req = resource_from(pt.req[:, p], int(pt.req_present[p]), L)
    prio = int(pt.priority[p])
    want = _tuples(entries, snap.want[p])

    def vreq(v):
        r = resource_from(bound.req[:, v], int(bound.req_present[v]), L)
        r.AllowedPodNumber = 0
        return r

    def more_important(a, b):
        ka = (-int(bound.priority[a]), int(bound.start_ns[a]), a)
        kb = (-int(bound.priority[b]), int(bound.start_ns[b]), b)
        return -1 if ka < kb else (1 if ka > kb else 0)

    cands = []
    for i in range(nt.n):
        node = Node(nt, i)
        if node.flags & 0x0F or not check_fit(sel, tol, node):
            continue
        if aff != 0xFFFFFFFF and not (int(aff_bits[aff, i // 32]) >> (i % 32)) & 1:
            continue
        left_keys = set(node.alloc.ScalarResources) & set(node.req.ScalarResources)
        if any(v != 0 and k not in left_keys for k, v in req.ScalarResources.items()):
            continue
        potential = [v for v in rows if int(bound.node[v]) == i and int(bound.priority[v]) < prio]
        if any(remove_pod(int(pt.gid[p]), int(bound.gid[v]), int(bound.flags[v]) & 1) != ALLOW for v in potential):
            continue
        c = copy.deepcopy(node)
        hp = set(used[i])
        for v in potential:
            _remove(c, vreq(v))
            hp -= _tuples(entries, ports[v])
        passes = lambda: _pod_fits(c, sel, tol, req) and not _conflict(hp | nom[i], want)
        if not passes():
            continue
        potential.sort(key=functools.cmp_to_key(more_important))
        violating = [v for v in potential if int(bound.flags[v]) & PDB_VIOLATING]
        others = [v for v in potential if not int(bound.flags[v]) & PDB_VIOLATING]
        victims, n_violating = [], 0
        for part, is_violating in ((violating, True), (others, False)):
            for v in part:   # reprievePod: addPod, the filters, removePod
                _add(c, vreq(v))
                hp |= _tuples(entries, ports[v])
                if not passes():
                    _remove(c, vreq(v))
                    hp -= _tuples(entries, ports[v])
                    victims.append(v)
                    n_violating += is_violating
        cands.append((i, victims, n_violating))
    node, victims = _pick(cands, bound)
    return node, victims, len(cands)


def _setup(snap, cols):
    (entries, used), want = cols
    entries = [tuple(int(x) for x in e) for e in np.asarray(entries).reshape(-1, 3)]
    s = snap.copy()
    s.want = np.asarray(want, np.uint64)
    return s, entries, [_tuples(entries, u) for u in used]


def preempt(snap, bound, cols, bound_ports, pods):
    """[(node or -1, [victim bound indices], n_candidates)] per pod."""
    s, entries, used = _setup(snap, cols)
    nom = [set() for _ in range(snap.nodes.n)]
    rows = list(range(bound.n))
    return [_preempt_one(s, bound, rows, entries, used, nom, bound_ports, int(p)) for p in pods]


def walk(snap, bound, cols, bound_ports, pods, gang=False):
    """[(node or -1, [victim bound indices], n_candidates, outcome)] per preemptor, and evicted_by [V]."""
    pods = [int(p) for p in pods]
    live, entries, used = _setup(snap, cols)
    nt, pt = live.nodes, live.pods
    nom = [set() for _ in range(nt.n)]
    evicted_by = [-1] * bound.n
    out = [None] * len(pods)
    for unit in _units(snap, pods, gang):
        saved = (nt.copy(), list(evicted_by), [set(u) for u in used], [set(m) for m in nom])
        failed = False
        for i in unit:
            rows = [v for v in range(bound.n) if evicted_by[v] < 0]
            node, victims, cand = _preempt_one(live, bound, rows, entries, used, nom, bound_ports, pods[i])
            if node < 0:
                failed = True
                out[i] = (-1, [], cand, NONE)
                continue
            out[i] = (node, victims, cand, NOMINATED)
            p = pods[i]
            for v in victims:            # NodeInfo.RemovePod
                evicted_by[v] = i
                used[node] -= _tuples(entries, bound_ports[v])
                for d in range(nt.lanes):
                    if d != 3 and (d < 4 or (int(bound.req_present[v]) >> d) & 1):
                        nt.requested[d, node] -= bound.req[d, v]
                nt.pod_count[node] -= 1
            for d in range(nt.lanes):     # the nominated pod: assume, and its ports on the nominated side
                if d != 3 and (d < 4 or (int(pt.req_present[p]) >> d) & 1):
                    nt.requested[d, node] += pt.req[d, p]
                    if d >= 4:
                        nt.req_present[node] |= np.uint32(1 << d)
            nt.pod_count[node] += 1
            nom[node] |= _tuples(entries, live.want[p])
        if gang and failed:
            live.nodes, evicted_by, used, nom = saved
            nt = live.nodes
            for i in unit:
                out[i] = (-1, [], out[i][2], ROLLED_BACK)
    return out, evicted_by
