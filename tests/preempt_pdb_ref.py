"""TEST INFRASTRUCTURE — the CPU restatement of bs_preempt with PodDisruptionBudget-violating bound pods
(include/bsched.h BS_BOUND_PDB_VIOLATING).

tests/preempt_pdb_ref.c mutates a one-node copy of each node and calls the oracle's fit predicate (bso_fit_eval) after
every removal and re-add, the way upstream's selectVictimsOnNode does, reprieving the violating potential victims
first, then picks the node by pickOneNodeForPreemption's criteria with the violation count first; OpenMP over the
preemptors.  It is compiled on first use into a library of its own, beside tests/native.py's library of the other
restatements, and takes the same tables and gives the same result type as tests/preempt_ref.py.
"""
from __future__ import annotations

import ctypes as C
import functools
import os
import subprocess

import numpy as np

import native
from oracle import oracle
from preempt_ref import PreemptResult, _Bound

_HERE = os.path.dirname(os.path.abspath(__file__))


@functools.cache
def _lib():
    so = oracle.build()
    out = os.path.join(native._out_dir().name, "libbs_preempt_pdb_ref.so")
    subprocess.check_call(["gcc", "-O2", "-std=c11", "-fPIC", "-Wall", "-Wextra", "-fopenmp", "-shared", "-o", out,
                           os.path.join(_HERE, "preempt_pdb_ref.c"), "-I" + os.path.join(os.path.dirname(_HERE), "oracle"),
                           so, "-Wl,-rpath," + os.path.dirname(so), "-lm"])
    oracle.lib()   # the oracle library first, so that its symbols resolve
    lib = C.CDLL(out)
    lib.bsp_preempt.restype = None
    lib.bsp_preempt.argtypes = [C.POINTER(oracle._Nodes), C.POINTER(oracle._Pods), C.POINTER(_Bound), C.c_void_p,
                                C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_int]
    return lib


def warm():
    """Compiles and loads the restatement (first use compiles it with gcc)."""
    _lib()


def preempt(snap, bound, pods=None, threads=0) -> PreemptResult:
    """bs_preempt's outputs for the pod indices `pods` (all pods when None); `bound` is a snapshot.BoundPodTable whose
    flags may carry BOUND_PDB_VIOLATING.  threads: OpenMP threads over the preemptors (<= 0: all)."""
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
    _lib().bsp_preempt(C.byref(nd), C.byref(pd), C.byref(b), idx.ctypes.data, n, node.ctypes.data, nv.ctypes.data,
                       cand.ctypes.data, vict.ctypes.data, vstride, int(threads))
    off = np.zeros(n + 1, np.uint32)
    off[1:] = np.cumsum(nv)
    victims = np.concatenate([vict[i, :nv[i]] for i in range(n)]).astype(np.uint32) if n else np.zeros(0, np.uint32)
    return PreemptResult(node, nv, cand, off, victims)
