"""TEST INFRASTRUCTURE — the CPU restatement of bs_remove_pod and bs_preempt (include/bsched.h).

tests/preempt_ref.c mutates a one-node copy of each node and calls the oracle's fit predicate (bso_fit_eval) after
every removal and re-add, the way upstream's selectVictimsOnNode does, with OpenMP over the preemptors.  It is
compiled into a temporary directory on first use, because the tree may be read-only, and linked against
oracle/libbs_oracle.so.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile
from dataclasses import dataclass

import numpy as np

from oracle import oracle

_HERE = os.path.dirname(os.path.abspath(__file__))
_ORACLE_DIR = os.path.join(os.path.dirname(_HERE), "oracle")
_lib_h = None

ALLOW, OFFLINE_ONLINE, NOT_FOUND, LOCKED, SAME_GROUP = range(5)
BOUND_GROUP_LOCKED = 0x01


class _Bound(C.Structure):
    _fields_ = [("n", C.c_uint32), ("lanes", C.c_uint32), ("node", C.c_void_p), ("req", C.c_void_p),
                ("req_present", C.c_void_p), ("gid", C.c_void_p), ("priority", C.c_void_p), ("start_ns", C.c_void_p),
                ("flags", C.c_void_p)]


def _lib():
    global _lib_h
    if _lib_h is None:
        so = oracle.build()
        out = os.path.join(tempfile.mkdtemp(prefix="preempt_ref_"), "libpreempt_ref.so")
        subprocess.check_call(["gcc", "-O2", "-std=c11", "-fPIC", "-Wall", "-Wextra", "-fopenmp", "-shared", "-o", out,
                               os.path.join(_HERE, "preempt_ref.c"), "-I" + _ORACLE_DIR, so,
                               "-Wl,-rpath," + os.path.dirname(so)])
        oracle.lib()   # the oracle library first, so that its symbols resolve
        lib = C.CDLL(out)
        lib.bsr_remove_pod.restype = C.c_int
        lib.bsr_remove_pod.argtypes = [C.c_int32, C.c_int32, C.c_uint8]
        lib.bsr_preempt.restype = None
        lib.bsr_preempt.argtypes = [C.POINTER(oracle._Nodes), C.POINTER(oracle._Pods), C.POINTER(_Bound), C.c_void_p,
                                    C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_int]
        _lib_h = lib
    return _lib_h


def remove_pod(gid_p: int, gid_v: int, flags_v: int) -> int:
    """core.PreemptRemovePod's verdict (ALLOW, OFFLINE_ONLINE, NOT_FOUND, LOCKED, SAME_GROUP)."""
    return int(_lib().bsr_remove_pod(int(gid_p), int(gid_v), int(flags_v)))


@dataclass
class PreemptResult:
    node: np.ndarray          # int32 [n]
    n_victims: np.ndarray     # uint32 [n]
    n_candidates: np.ndarray  # uint32 [n]
    victim_offset: np.ndarray # uint32 [n + 1]
    victims: np.ndarray       # uint32 [total]

    def victims_of(self, i):
        return self.victims[self.victim_offset[i]:self.victim_offset[i + 1]].tolist()


def warm():
    """Compiles and loads the restatement (first use compiles it with gcc)."""
    _lib()


def preempt(snap, bound, pods=None, threads=0) -> PreemptResult:
    """bs_preempt's outputs for the pod indices `pods` (all pods when None); `bound` is a snapshot.BoundPodTable.
    threads: OpenMP threads over the preemptors (<= 0: all)."""
    nt, pt = snap.nodes, snap.pods
    idx = np.ascontiguousarray(np.arange(pt.n) if pods is None else pods, dtype=np.uint32)
    n = len(idx)
    counts = np.bincount(bound.node.astype(np.int64), minlength=nt.n) if bound.n else np.zeros(nt.n, np.int64)
    vstride = max(1, int(counts.max()) if nt.n else 1)
    node = np.zeros(n, np.int32)
    nv = np.zeros(n, np.uint32)
    cand = np.zeros(n, np.uint32)
    vict = np.zeros((max(n, 1), vstride), np.uint32)
    nd, pd = oracle._nodes(nt, getattr(snap, "aff_bits", None)), oracle._pods(pt)
    b = _Bound(bound.n, bound.lanes, *(bound.node.ctypes.data, bound.req.ctypes.data, bound.req_present.ctypes.data,
                                       bound.gid.ctypes.data, bound.priority.ctypes.data, bound.start_ns.ctypes.data,
                                       bound.flags.ctypes.data))
    _lib().bsr_preempt(C.byref(nd), C.byref(pd), C.byref(b), idx.ctypes.data, n, node.ctypes.data, nv.ctypes.data,
                       cand.ctypes.data, vict.ctypes.data, vstride, int(threads))
    off = np.zeros(n + 1, np.uint32)
    off[1:] = np.cumsum(nv)
    victims = np.concatenate([vict[i, :nv[i]] for i in range(n)]).astype(np.uint32) if n else np.zeros(0, np.uint32)
    return PreemptResult(node, nv, cand, off, victims)
