"""TEST INFRASTRUCTURE — the walks (bs_replay, bs_replay_priority) with the MatchInterPodAffinity filter on, restated
on the packed columns: tests/interpod_walk_ref.c's hook pair around any of the choosers of bsr_replay_choose (first
fit, priority, ratio, locality), optionally with tests/host_ports_ref.c's pair in between.  The C file is compiled on
first use into a library of its own in tests/native.py's temporary directory.
"""
from __future__ import annotations

import ctypes as C
import functools
import os
import subprocess

import numpy as np

import host_ports_ref as hr
import native

_HERE = os.path.dirname(os.path.abspath(__file__))


class _Classes(C.Structure):
    _fields_ = [("off", C.c_void_p), ("term", C.c_void_p), ("own", C.c_void_p), ("match", C.c_void_p)]


class _Ctx(C.Structure):
    _fields_ = [("inner", C.c_void_p), ("inner_assumed", C.c_void_p), ("inner_ctx", C.c_void_p),
                ("n_nodes", C.c_uint32), ("topo", C.c_void_p), ("term_key", C.c_void_p), ("n_bound", C.c_uint32),
                ("bound_node", C.c_void_p), ("bound_class", C.c_void_p), ("bound", _Classes),
                ("pod_class", C.c_void_p), ("p_off", C.c_void_p), ("p_term", C.c_void_p), ("p_role", C.c_void_p),
                ("p_self", C.c_void_p), ("placed_class", C.c_void_p), ("placed", _Classes),
                ("assumed_pod", C.c_void_p), ("assumed_node", C.c_void_p), ("n_assumed", C.c_uint32)]


class _LocCtx(C.Structure):   # tests/locality_priority_ref.c bsr_locality_ctx
    _fields_ = [("node_nz", C.c_void_p), ("pod_nz", C.c_void_p), ("w_least", C.c_uint32), ("w_most", C.c_uint32),
                ("w_balanced", C.c_uint32), ("s", C.c_void_p), ("q", C.c_void_p)]


@functools.cache
def _lib():
    out = os.path.join(native._out_dir().name, "libbs_interpod_walk_ref.so")
    subprocess.check_call(["gcc", "-O2", "-std=c11", "-fPIC", "-Wall", "-Wextra", "-shared", "-o", out,
                           os.path.join(_HERE, "interpod_walk_ref.c"),
                           "-I" + os.path.join(os.path.dirname(_HERE), "oracle"), "-I" + _HERE])
    return C.CDLL(out)


def _fn(lib, name):
    return C.cast(getattr(lib, name), C.c_void_p).value


def _classes(cl, keep):
    off = np.ascontiguousarray(cl[0], np.uint32).reshape(-1)
    term = np.ascontiguousarray(cl[1], np.uint32).reshape(-1)
    own = np.ascontiguousarray(cl[2], np.int32).reshape(-1)
    match = np.ascontiguousarray(cl[3], np.uint8).reshape(-1)
    keep += [off, term, own, match]
    return _Classes(off.ctypes.data, term.ctypes.data, own.ctypes.data, match.ctypes.data)


def replay(snap, cols, placed, queue=None, nz=None, weights=(1, 0, 1), ratio=None, loc=None, lw=(0, 0), hp=None):
    """The walk with the filter on, on COPIES of the tables.  cols = (node, pods) as Engine.upload_interpod_filter
    takes them, placed = (pod_class, classes) as Engine.upload_interpod_placed takes them.  The node choice: first fit
    (nz None), bs_replay_priority's chooser (nz = (node_nz, pod_nz)), with the ratio term (ratio as
    ratio_priority_ref.setting takes it) and with the locality terms (loc = snapshot.node_locality's columns, lw their
    weights).  hp: host_ports_ref's columns, whose filter runs inside this one.  Returns (prefilter, node, ready,
    snap_after, live non-zero column [2, N] or None, live used masks [N] or None)."""
    import locality_priority_ref as lr
    import ratio_priority_ref as rr
    import replay_priority_ref as rpr
    ref = rpr._lib()
    keep = []
    N, P = snap.nodes.n, snap.pods.n
    nz_live = hp_live = None
    if nz is None:
        inner, inner_assumed, inner_ctx = _fn(ref, "bsr_first_fit"), None, None
    else:
        nz_live = np.array(nz[0], dtype=np.int64).reshape(2, N)
        pod_nz = np.ascontiguousarray(nz[1], dtype=np.int64).reshape(2, P)
        keep.append(pod_nz)
        if loc is not None:
            r = ratio if ratio is not None else lr.NO_RATIO
            lanes = list(r[2]) + [0] * (snap.nodes.lanes - len(r[2]))
            setting = rr.setting(r[0], r[1], lanes, *r[3:])
            lcols = lr.Columns(loc, N, lw)
            keep += [setting, lcols]
            ictx = _LocCtx(nz_live.ctypes.data, pod_nz.ctypes.data, *weights, C.addressof(setting),
                           C.addressof(lcols.q))
            inner, inner_assumed = _fn(lr._lib(), "bsr_locality_choose"), _fn(ref, "bsr_priority_assumed")
        elif ratio is not None:
            rr._lib()
            setting = rr.setting(*ratio)
            keep.append(setting)
            ictx = hr._RatioCtx(nz_live.ctypes.data, pod_nz.ctypes.data, *weights, C.addressof(setting))
            inner, inner_assumed = _fn(ref, "bsr_ratio_choose"), _fn(ref, "bsr_ratio_assumed")
        else:
            ictx = hr._PriorityCtx(nz_live.ctypes.data, pod_nz.ctypes.data, *weights)
            inner, inner_assumed = _fn(ref, "bsr_priority_choose"), _fn(ref, "bsr_priority_assumed")
        keep.append(ictx)
        inner_ctx = C.addressof(ictx)
    if hp is not None:
        (entries, used), want = hp
        d, dkeep = hr._dict(entries)
        hp_live = np.array(used, dtype=np.uint64)
        want = np.ascontiguousarray(want, dtype=np.uint64)
        hctx = hr._Ctx(inner, inner_assumed, inner_ctx, d, hp_live.ctypes.data, want.ctypes.data)
        keep += [dkeep, want, hctx]
        hl = hr._lib()
        inner, inner_assumed, inner_ctx = _fn(hl, "bsr_hp_choose"), _fn(hl, "bsr_hp_assumed"), C.addressof(hctx)
    (nv, topo, tkey, bnode, bcls, bcl), (pcls, (poff, pterm, prole, pself)) = cols
    u32 = lambda a: np.ascontiguousarray(a, dtype=np.uint32).reshape(-1)
    u8 = lambda a: np.ascontiguousarray(a, dtype=np.uint8).reshape(-1)
    cap = max(P if queue is None else len(queue), 1)   # every queue position assumes at most one pod
    arr = [u32(topo) if len(nv) else np.zeros(1, np.uint32), u32(tkey), u32(bnode), u32(bcls), u32(pcls), u32(poff),
           u32(pterm), u8(prole), u8(pself), u32(placed[0]), np.zeros(cap, np.uint32), np.zeros(cap, np.uint32)]
    keep += arr
    a = [x.ctypes.data for x in arr]
    ctx = _Ctx(inner, inner_assumed, inner_ctx, N, a[0], a[1], len(arr[2]), a[2], a[3], _classes(bcl, keep),
               *a[4:9], a[9], _classes(placed[1], keep), a[10], a[11], 0)
    lib = _lib()
    choose, assumed = _fn(lib, "bsr_ipw_choose"), _fn(lib, "bsr_ipw_assumed")
    pf, node, ready, after = rpr._walk(snap, queue, lambda *x: ref.bsr_replay_choose(*x, choose, assumed,
                                                                                      C.addressof(ctx)))
    return pf, node, ready, after, nz_live, hp_live
