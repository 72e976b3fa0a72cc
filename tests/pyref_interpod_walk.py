"""TEST INFRASTRUCTURE — the walks with the MatchInterPodAffinity filter restated from objects, and the placed classes
of the pending pods (include/bsched.h bs_upload_pod_interpod_placed) packed from the same objects.

walk() is the oracle's pod-at-a-time walk (tests/replay_priority_ref.c bsr_replay_choose, first fit) whose chooser asks
pyref_interpod_filter.verdict() for every node, with the pods assumed so far simply appended to the existing pods.
placed() resolves the pending pods against pyref_interpod_filter.pack()'s dictionary, whose term ids it recomputes in
pack's order: the bound pods' anti-affinity terms, then per pending pod its affinity terms and its anti-affinity terms.
"""
from __future__ import annotations

import ctypes as C
import dataclasses

import numpy as np

import pyref_interpod_filter as pyf
from oracle import oracle

UNSCHEDULABLE = 0x04   # BSO_NODE_UNSCHEDULABLE


def _dictionary(nodes, existing, pending):
    """(owned, aff, anti): the bound pods' distinct anti-affinity terms [(term id, Term with its owner's namespaces)],
    and per pending pod its affinity and anti-affinity term ids, as pack() numbers them."""
    bound = [e for e in existing if e.node in nodes]
    n = 0
    owned = {}
    for e in bound:
        for w in e.anti:
            ident = (tuple(sorted(w.namespaces or [e.ns])), repr(w.selector), w.key)
            if ident not in owned:
                owned[ident] = (n, pyf.Term(w.selector, w.key, list(w.namespaces or [e.ns])))
                n += 1
    aff, anti = [], []
    for p in pending:
        aff.append(list(range(n, n + len(p.affinity))))
        n += len(p.affinity)
        anti.append(list(range(n, n + len(p.anti))))
        n += len(p.anti)
    return list(owned.values()), aff, anti


def placed(nodes, existing, pending):
    """(pod_class [P], (class_offset, term, own int32, match uint8)) over pack()'s dictionary: own 1 on the pod's own
    anti-affinity terms; match 1 on the bound pods' anti-affinity terms it matches, on every term of each pending pod's
    affinity set it matches as a whole (its own set included) and on each pending pod's anti-affinity terms it
    matches."""
    owned, aff, anti = _dictionary(nodes, existing, pending)
    pod_class, off, term, own, match = [], [0], [], [], []
    for i, p in enumerate(pending):
        ent = {}
        for t in anti[i]:
            ent.setdefault(t, [0, 0])[0] = 1
        for t, w in owned:
            if pyf.pod_matches_term(p, w, p.ns):   # w carries its owner's namespaces
                ent.setdefault(t, [0, 0])[1] = 1
        for j, r in enumerate(pending):
            if r.affinity and all(pyf.pod_matches_term(p, x, r.ns) for x in r.affinity):
                for t in aff[j]:
                    ent.setdefault(t, [0, 0])[1] = 1
            for t, u in zip(anti[j], r.anti):
                if pyf.pod_matches_term(p, u, r.ns):
                    ent.setdefault(t, [0, 0])[1] = 1
        if not ent:
            pod_class.append(pyf.IPF_NONE)
            continue
        pod_class.append(len(off) - 1)
        for t in sorted(ent):
            term.append(t); own.append(ent[t][0]); match.append(ent[t][1])
        off.append(len(term))
    return (np.array(pod_class, np.uint32), (np.array(off, np.uint32), np.array(term, np.uint32),
                                             np.array(own, np.int32), np.array(match, np.uint8)))


_CHOOSE = C.CFUNCTYPE(C.c_int32, C.c_void_p, C.POINTER(oracle._Nodes), C.POINTER(oracle._Pods), C.c_uint32)
_ASSUMED = C.CFUNCTYPE(None, C.c_void_p, C.POINTER(oracle._Nodes), C.POINTER(oracle._Pods), C.c_uint32, C.c_uint32)


def walk(snap, nodes, existing, pending, queue=None):
    """The first-fit walk on COPIES of the tables with the filter decided from objects: pending[p] is pod p of the
    table, nodes (name -> labels) lists the table's nodes in order.  Returns (prefilter, node, ready, snap_after)."""
    import replay_priority_ref as rpr
    ref = rpr._lib()
    names = list(nodes)
    first_fit = C.cast(ref.bsr_first_fit, C.CFUNCTYPE(C.c_int32, C.c_void_p, C.POINTER(oracle._Nodes),
                                                       C.POINTER(oracle._Pods), C.c_uint32))
    assumed = []

    def choose(ctx, nd, pd, p):
        flags = nd.contents.flags
        saved = [flags[n] for n in range(len(names))]
        ex = list(existing) + assumed
        for n, name in enumerate(names):
            if pyf.verdict(pending[p], name, nodes, ex) is not None:
                flags[n] = flags[n] | UNSCHEDULABLE
        r = first_fit(None, nd, pd, p)
        for n in range(len(names)):
            flags[n] = saved[n]
        return r

    def on_assumed(ctx, nd, pd, p, n):
        assumed.append(dataclasses.replace(pending[p], node=names[n]))

    cb_choose, cb_assumed = _CHOOSE(choose), _ASSUMED(on_assumed)
    return rpr._walk(snap, queue, lambda *a: ref.bsr_replay_choose(*a, C.cast(cb_choose, C.c_void_p),
                                                                   C.cast(cb_assumed, C.c_void_p), None))
