"""TEST INFRASTRUCTURE, NOT PRODUCT — ctypes binding of oracle/libbs_oracle.so.

The oracle is the CPU restatement of pkg/scheduler/core/core.go (see bs_oracle.h).
Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
legs may import this module.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from dataclasses import dataclass

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libbs_oracle.so")
MAX_LANES = 16


def build(force: bool = False) -> str:
    src = [os.path.join(_HERE, f) for f in ("bs_oracle.c", "bs_gang.c", "bs_oracle.h")]
    if force or not os.path.exists(_LIB_PATH) or any(
            os.path.getmtime(s) > os.path.getmtime(_LIB_PATH) for s in src if os.path.exists(s)):
        subprocess.check_call(["make", "-C", _HERE, "-s", "libbs_oracle.so"])
    return _LIB_PATH


class _Resource(C.Structure):
    _fields_ = [("v", C.c_int64 * MAX_LANES), ("present", C.c_uint32)]


def _p(t):
    return C.POINTER(t)


class _Nodes(C.Structure):
    _fields_ = [("n", C.c_uint32), ("lanes", C.c_uint32), ("alloc", _p(C.c_int64)),
                ("requested", _p(C.c_int64)), ("pod_count", _p(C.c_int32)),
                ("alloc_present", _p(C.c_uint32)), ("req_present", _p(C.c_uint32)),
                ("label_mask", _p(C.c_uint64)), ("taint_mask", _p(C.c_uint64)), ("flags", _p(C.c_uint8)),
                ("n_aff", C.c_uint32), ("aff_bits", _p(C.c_uint32))]


class _Pods(C.Structure):
    _fields_ = [("n", C.c_uint32), ("lanes", C.c_uint32), ("req", _p(C.c_int64)),
                ("req_present", _p(C.c_uint32)), ("gid", _p(C.c_int32)), ("sel_mask", _p(C.c_uint64)),
                ("tol_mask", _p(C.c_uint64)), ("priority", _p(C.c_int32)), ("ts_ns", _p(C.c_int64)),
                ("flags", _p(C.c_uint8)), ("aff_class", _p(C.c_uint32))]


class _Groups(C.Structure):
    _fields_ = [("n", C.c_uint32), ("lanes", C.c_uint32), ("min_member", _p(C.c_uint32)),
                ("scheduled", _p(C.c_uint32)), ("matched", _p(C.c_uint32)), ("flags", _p(C.c_uint8)),
                ("min_res", _p(C.c_int64)), ("min_res_present", _p(C.c_uint32)),
                ("rep_sel", _p(C.c_uint64)), ("rep_tol", _p(C.c_uint64)), ("creation_ns", _p(C.c_int64)),
                ("name_rank", _p(C.c_uint32)), ("rep_aff", _p(C.c_uint32))]


class _Results(C.Structure):
    _fields_ = [("prefilter", _p(C.c_uint8)), ("feasible_count", _p(C.c_uint32)),
                ("best_node", _p(C.c_int32)), ("best_score", _p(C.c_int64)), ("admit", _p(C.c_uint8)),
                ("admit_bitmap", _p(C.c_uint32)), ("new_denied", _p(C.c_uint8)), ("order", _p(C.c_uint32)),
                ("rank", _p(C.c_uint32)), ("filter_bitmap", _p(C.c_uint32)), ("filter_code", _p(C.c_uint8)),
                ("fit_bitmap", _p(C.c_uint32)), ("score", _p(C.c_int64)),
                ("max_group", C.c_int32), ("max_finished", C.c_uint32), ("ref_panic", C.c_int32)]


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(_LIB_PATH)
        _lib.bso_scale.restype = C.c_int64
        _lib.bso_scale.argtypes = [C.c_int64, C.c_float]
        _lib.bso_permit_ready.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32]
        _lib.bso_compare_cluster.argtypes = [_p(_Nodes), C.c_uint64, C.c_uint64, C.c_uint32, _p(_Resource), C.c_float]
        _lib.bso_single_node_resource.argtypes = [_p(_Nodes), C.c_uint32, C.c_uint64, C.c_uint64, C.c_uint32,
                                                  C.c_float, _p(_Resource)]
        _lib.bso_compute_cluster.argtypes = [_p(_Nodes), C.c_uint64, C.c_uint64, C.c_uint32, _p(_Resource)]
        _lib.bso_pre_allocated.argtypes = [_p(_Groups), C.c_uint32, C.c_int64, _p(_Resource)]
        _lib.bso_fit_eval.argtypes = [_p(_Nodes), _p(_Pods), C.c_uint32, C.c_uint32, _p(C.c_int64)]
        _lib.bso_compare.argtypes = [_p(_Pods), _p(_Groups), C.c_uint32, C.c_uint32]
        _lib.bso_find_max_pg.argtypes = [_p(_Groups), _p(C.c_uint32), _p(C.c_int)]
        _lib.bso_round.argtypes = [_p(_Nodes), _p(_Pods), _p(_Groups), _p(_Results), C.c_int, C.c_int]
    return _lib


def _ptr(a, t):
    return a.ctypes.data_as(_p(t))


AFF_NONE = 0xFFFFFFFF


def _nodes(nt, aff_bits=None):
    """aff_bits: Snapshot.aff_bits ([n_aff, ceil(N/32)] uint32) or None."""
    if aff_bits is not None:
        assert aff_bits.dtype == np.uint32 and aff_bits.flags["C_CONTIGUOUS"] and aff_bits.shape[1] == (nt.n + 31) // 32
    return _Nodes(nt.n, nt.lanes, _ptr(nt.alloc, C.c_int64), _ptr(nt.requested, C.c_int64),
                  _ptr(nt.pod_count, C.c_int32), _ptr(nt.alloc_present, C.c_uint32),
                  _ptr(nt.req_present, C.c_uint32), _ptr(nt.label_mask, C.c_uint64),
                  _ptr(nt.taint_mask, C.c_uint64), _ptr(nt.flags, C.c_uint8),
                  0 if aff_bits is None else aff_bits.shape[0], None if aff_bits is None else _ptr(aff_bits, C.c_uint32))


def _pods(pt):
    aff = getattr(pt, "aff_class", None)
    return _Pods(pt.n, pt.lanes, _ptr(pt.req, C.c_int64), _ptr(pt.req_present, C.c_uint32),
                 _ptr(pt.gid, C.c_int32), _ptr(pt.sel_mask, C.c_uint64), _ptr(pt.tol_mask, C.c_uint64),
                 _ptr(pt.priority, C.c_int32), _ptr(pt.ts_ns, C.c_int64), _ptr(pt.flags, C.c_uint8),
                 None if aff is None else _ptr(aff, C.c_uint32))


def _groups(gt):
    return _Groups(gt.n, gt.lanes, _ptr(gt.min_member, C.c_uint32), _ptr(gt.scheduled, C.c_uint32),
                   _ptr(gt.matched, C.c_uint32), _ptr(gt.flags, C.c_uint8), _ptr(gt.min_res, C.c_int64),
                   _ptr(gt.min_res_present, C.c_uint32), _ptr(gt.rep_sel, C.c_uint64),
                   _ptr(gt.rep_tol, C.c_uint64), _ptr(gt.creation_ns, C.c_int64),
                   _ptr(gt.name_rank, C.c_uint32),
                   None if getattr(gt, "rep_aff", None) is None else _ptr(gt.rep_aff, C.c_uint32))


def _res_from(vals, present, lanes):
    r = _Resource()
    for d in range(lanes):
        r.v[d] = int(vals[d])
    r.present = int(present)
    return r


def scale(alloc: int, percent: float) -> int:
    return lib().bso_scale(int(alloc), C.c_float(percent))


def permit_ready(matched: int, min_member: int, scheduled: int) -> bool:
    return bool(lib().bso_permit_ready(matched, min_member, scheduled))


def single_node_resource(nt, i, sel, tol, percent, aff=AFF_NONE, aff_bits=None):
    r = _Resource()
    nd = _nodes(nt, aff_bits)
    lib().bso_single_node_resource(C.byref(nd), i, int(sel), int(tol), int(aff), C.c_float(percent), C.byref(r))
    return np.array(r.v[:nt.lanes], dtype=np.int64), int(r.present)


def node_left(nt, sel, tol, percent):
    """singleNodeResource over every node -> (left[L,N], present[N])."""
    left = np.zeros((nt.lanes, nt.n), np.int64)
    pres = np.zeros(nt.n, np.uint32)
    nd = _nodes(nt)
    r = _Resource()
    f = lib().bso_single_node_resource
    for i in range(nt.n):
        f(C.byref(nd), i, int(sel), int(tol), AFF_NONE, C.c_float(percent), C.byref(r))
        left[:, i] = r.v[:nt.lanes]
        pres[i] = r.present
    return left, pres


def compare_cluster(nt, sel, tol, need, need_present, percent, aff=AFF_NONE, aff_bits=None) -> bool:
    nd = _nodes(nt, aff_bits)
    r = _res_from(need, need_present, nt.lanes)
    return bool(lib().bso_compare_cluster(C.byref(nd), int(sel), int(tol), int(aff), C.byref(r), C.c_float(percent)))


def compute_cluster(nt, sel, tol):
    nd = _nodes(nt)
    r = _Resource()
    lib().bso_compute_cluster(C.byref(nd), int(sel), int(tol), AFF_NONE, C.byref(r))
    return np.array(r.v[:nt.lanes], dtype=np.int64), int(r.present)


def pre_allocated(gt, g, matched):
    gr = _groups(gt)
    r = _Resource()
    lib().bso_pre_allocated(C.byref(gr), g, int(matched), C.byref(r))
    return np.array(r.v[:gt.lanes], dtype=np.int64), int(r.present)


def fit_eval(nt, pt, p, n):
    nd, pd = _nodes(nt), _pods(pt)
    s = C.c_int64()
    f = lib().bso_fit_eval(C.byref(nd), C.byref(pd), p, n, C.byref(s))
    return bool(f), int(s.value)


def compare(pt, gt, a, b) -> bool:
    pd, gr = _pods(pt), _groups(gt)
    return bool(lib().bso_compare(C.byref(pd), C.byref(gr), a, b))


def find_max_pg(gt):
    gr = _groups(gt)
    mf, pn = C.c_uint32(), C.c_int()
    m = lib().bso_find_max_pg(C.byref(gr), C.byref(mf), C.byref(pn))
    return m, int(mf.value), bool(pn.value)


@dataclass
class RoundResult:
    prefilter: np.ndarray
    feasible_count: np.ndarray
    best_node: np.ndarray
    best_score: np.ndarray
    admit: np.ndarray
    admit_bitmap: np.ndarray
    new_denied: np.ndarray
    order: np.ndarray
    rank: np.ndarray
    fit_bitmap: np.ndarray | None
    score: np.ndarray | None
    filter_bitmap: np.ndarray | None
    filter_code: np.ndarray | None
    max_group: int
    max_finished: int
    ref_panic: bool


def round(snap, want_bitmap=True, want_score=False, faithful=False, threads=0, want_sort=True,
          want_filter=False) -> RoundResult:
    """One snapshot round (DESIGN.md 'Round semantics') on the CPU oracle."""
    nt, pt, gt = snap.nodes, snap.pods, snap.groups
    P, N, G = pt.n, nt.n, gt.n
    words = (N + 31) // 32
    r = RoundResult(np.zeros(P, np.uint8), np.zeros(P, np.uint32), np.zeros(P, np.int32),
                    np.zeros(P, np.int64), np.zeros(G, np.uint8), np.zeros((G + 31) // 32, np.uint32),
                    np.zeros(G, np.uint8), np.zeros(P, np.uint32), np.zeros(P, np.uint32),
                    np.zeros((P, words), np.uint32) if want_bitmap else None,
                    np.zeros((P, N), np.int64) if want_score else None,
                    np.zeros((P, words), np.uint32) if want_filter else None,
                    np.zeros(P, np.uint8) if want_filter else None, -1, 0, False)
    res = _Results(_ptr(r.prefilter, C.c_uint8), _ptr(r.feasible_count, C.c_uint32),
                   _ptr(r.best_node, C.c_int32), _ptr(r.best_score, C.c_int64), _ptr(r.admit, C.c_uint8),
                   _ptr(r.admit_bitmap, C.c_uint32), _ptr(r.new_denied, C.c_uint8),
                   _ptr(r.order, C.c_uint32) if want_sort else None,
                   _ptr(r.rank, C.c_uint32) if want_sort else None,
                   _ptr(r.filter_bitmap, C.c_uint32) if want_filter else None,
                   _ptr(r.filter_code, C.c_uint8) if want_filter else None,
                   _ptr(r.fit_bitmap, C.c_uint32) if want_bitmap else None,
                   _ptr(r.score, C.c_int64) if want_score else None, -1, 0, 0)
    nd, pd, gr = _nodes(nt, getattr(snap, "aff_bits", None)), _pods(pt), _groups(gt)
    rc = lib().bso_round(C.byref(nd), C.byref(pd), C.byref(gr), C.byref(res), int(faithful), int(threads))
    if rc < 0:
        raise MemoryError("oracle round failed")
    r.max_group, r.max_finished, r.ref_panic = int(res.max_group), int(res.max_finished), bool(res.ref_panic)
    return r


def replay(snap, queue=None, panic=False):
    """Sequential pod-at-a-time replay on COPIES of the tables; returns (prefilter, node, ready, snap_after) and, with
    panic=True, a fifth value: the first queue position where findMaxPG would divide by MinMember == 0 (the reference
    panics there; bs_replay returns BS_E_REF_PANIC), or None."""
    s = snap.copy()
    nt, pt, gt = s.nodes, s.pods, s.groups
    q = np.ascontiguousarray(np.arange(pt.n) if queue is None else queue, dtype=np.uint32)
    pf = np.zeros(len(q), np.uint8)
    node = np.zeros(len(q), np.int32)
    ready = np.zeros(len(q), np.uint8)
    if pt.aff_class is not None and gt.rep_aff is None:
        gt.rep_aff = np.full(gt.n, AFF_NONE, np.uint32)   # the walk records the first pod's class here
    nd, pd, gr = _nodes(nt, getattr(s, "aff_bits", None)), _pods(pt), _groups(gt)
    f = lib().bso_replay
    f.restype = C.c_int
    f.argtypes = [_p(_Nodes), _p(_Pods), _p(_Groups), _p(C.c_uint32), C.c_uint32, _p(C.c_uint8),
                  _p(C.c_int32), _p(C.c_uint8)]
    at = f(C.byref(nd), C.byref(pd), C.byref(gr), _ptr(q, C.c_uint32), len(q), _ptr(pf, C.c_uint8),
           _ptr(node, C.c_int32), _ptr(ready, C.c_uint8))
    if panic:
        return pf, node, ready, s, (None if at < 0 else int(at))
    return pf, node, ready, s


def max_threads() -> int:
    return int(lib().bso_max_threads())


class Gang:
    """CPU model of the state around Permit (oracle/bs_gang.c): MatchedPodNodes / PodNameUIDs with TTLs, the
    deny and permitted caches, the eviction callback and the Allow loop."""

    def __init__(self, n_groups: int):
        L = lib()
        L.bso_gang_new.restype = C.c_void_p
        L.bso_gang_new.argtypes = [C.c_uint32]
        L.bso_gang_free.argtypes = [C.c_void_p]
        L.bso_permit_step.argtypes = [C.c_void_p, C.c_uint32, C.c_uint64, C.c_uint64, C.c_uint32, C.c_int64, C.c_int64,
                                      C.c_uint32, C.c_uint32]
        L.bso_expire.restype = C.c_uint32
        L.bso_expire.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32,
                                 _p(C.c_uint32)]
        L.bso_allow_list.restype = C.c_uint32
        L.bso_allow_list.argtypes = [C.c_void_p, C.c_uint32, C.c_int64, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p,
                                     C.c_uint32]
        L.bso_gang_matched.restype = C.c_uint32
        L.bso_gang_matched.argtypes = [C.c_void_p, C.c_uint32, C.c_int64]
        L.bso_gang_scheduled.argtypes = [C.c_void_p, C.c_uint32]
        L.bso_gang_denied.argtypes = [C.c_void_p, C.c_uint32, C.c_int64]
        L.bso_gang_deny.argtypes = [C.c_void_p, C.c_uint32, C.c_int64]
        L.bso_gang_permitted.argtypes = [C.c_void_p, C.c_uint64, C.c_int64]
        L.bso_gang_mark_permitted.argtypes = [C.c_void_p, C.c_uint64, C.c_int64]
        self.L, self.n = L, n_groups
        self.h = L.bso_gang_new(n_groups)

    def __del__(self):
        if getattr(self, "h", None):
            self.L.bso_gang_free(self.h)
            self.h = None

    def permit(self, g, uid, name, node, now, wait_ns, min_member, scheduled) -> bool:
        return bool(self.L.bso_permit_step(self.h, g, uid, name, node, now, wait_ns, min_member, scheduled))

    def expire(self, now, cap=4096):
        rg, ru = np.zeros(cap, np.uint32), np.zeros(cap, np.uint64)
        ev = np.zeros(max(self.n, 1), np.uint32)
        ne = C.c_uint32()
        n = self.L.bso_expire(self.h, now, rg.ctypes.data, ru.ctypes.data, cap, ev.ctypes.data, len(ev), C.byref(ne))
        return list(zip(rg[:n].tolist(), ru[:n].tolist())), ev[:ne.value].tolist()

    def allow_list(self, g, now, min_member, scheduled, cap=4096):
        u, nd = np.zeros(cap, np.uint64), np.zeros(cap, np.uint32)
        n = self.L.bso_allow_list(self.h, g, now, min_member, scheduled, u.ctypes.data, nd.ctypes.data, cap)
        return u[:n].tolist(), nd[:n].tolist()

    def matched(self, g, now):
        return int(self.L.bso_gang_matched(self.h, g, now))

    def scheduled(self, g):
        return bool(self.L.bso_gang_scheduled(self.h, g))

    def denied(self, g, now):
        return bool(self.L.bso_gang_denied(self.h, g, now))

    def deny(self, g, now):
        self.L.bso_gang_deny(self.h, g, now)

    def permitted(self, uid, now):
        return bool(self.L.bso_gang_permitted(self.h, uid, now))

    def mark_permitted(self, uid, now):
        self.L.bso_gang_mark_permitted(self.h, uid, now)
