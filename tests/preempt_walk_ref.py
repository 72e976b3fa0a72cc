"""TEST INFRASTRUCTURE — the CPU restatement of bs_preempt_walk (include/bsched.h).

tests/preempt_walk_ref.c walks the preemptors in list order, each one tests/preempt_pdb_ref.c's single-pod preemption
on a master node state and the bound pods not yet evicted; the victims leave by preempt_pdb_ref.c's apply() and the
preemptor is added by the oracle's assume step; a failed gang unit is undone from a saved copy.

It is compiled on first use into a library of its own, in tests/native.py's build directory and against the same
oracle library, the way tests/preempt_pdb_ref.py builds preempt_pdb_ref.c.  The walk reuses that file's static
helpers (copy_node, apply) and its single-pod bsp_preempt by including it, and preempt_pdb_ref.c is not among
native.py's shared sources, so the walk is built beside it rather than into the shared library.
"""
from __future__ import annotations

import ctypes as C
import functools
import os
import subprocess
from dataclasses import dataclass

import numpy as np

import native
from oracle import oracle
from preempt_ref import PreemptResult, _Bound

_HERE = os.path.dirname(os.path.abspath(__file__))
NONE, NOMINATED, ROLLED_BACK = range(3)   # BS_WALK_*


@functools.cache
def _lib():
    so = oracle.build()
    out = os.path.join(native._out_dir().name, "libbs_preempt_walk_ref.so")
    subprocess.check_call(["gcc", "-O2", "-std=c11", "-fPIC", "-Wall", "-Wextra", "-fopenmp", "-shared", "-o", out,
                           os.path.join(_HERE, "preempt_walk_ref.c"), "-I" + _HERE,
                           "-I" + os.path.join(os.path.dirname(_HERE), "oracle"), so,
                           "-Wl,-rpath," + os.path.dirname(so), "-lm"])
    oracle.lib()   # the oracle library first, so that its symbols resolve
    lib = C.CDLL(out)
    lib.bsw_walk.restype = C.c_uint32
    lib.bsw_walk.argtypes = [C.POINTER(oracle._Nodes), C.POINTER(oracle._Pods), C.POINTER(_Bound), C.c_void_p,
                             C.c_uint32, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                             C.c_void_p, C.c_void_p]
    return lib


@dataclass
class WalkResult(PreemptResult):
    outcome: np.ndarray = None      # uint32 [n] NONE / NOMINATED / ROLLED_BACK
    evicted_by: np.ndarray = None   # int32 [V]


def units_last(snap, pods, gang):
    """unit_last[i]: step i closes its unit.  With gang, a run of preemptors of one group (0 <= gid < n_groups) is one
    unit; any other gid names no group of the table and makes a unit of one."""
    gid = snap.pods.gid[np.asarray(pods, np.int64)] if len(pods) else np.zeros(0, np.int32)
    last = np.ones(len(pods), np.uint8)
    if gang:
        for i in range(len(pods) - 1):
            if 0 <= gid[i] < snap.groups.n and gid[i] == gid[i + 1]:
                last[i] = 0
    return last


def walk(snap, bound, pods, gang=False) -> WalkResult:
    """bs_preempt_walk's outputs for the pod indices `pods` in list order (the caller keeps the engine's list rules)."""
    nt, pt = snap.nodes, snap.pods
    idx = np.ascontiguousarray(pods, dtype=np.uint32)
    n, V = len(idx), bound.n
    node, nv, cand, outcome = (np.zeros(n, np.int32), np.zeros(n, np.uint32), np.zeros(n, np.uint32),
                               np.zeros(n, np.uint32))
    vict = np.zeros(max(V, 1), np.uint32)
    evby = np.zeros(max(V, 1), np.int32)
    last = units_last(snap, idx, gang)
    nd, pd = oracle._nodes(nt, getattr(snap, "aff_bits", None)), oracle._pods(pt)
    b = _Bound(bound.n, bound.lanes, *(bound.node.ctypes.data, bound.req.ctypes.data, bound.req_present.ctypes.data,
                                       bound.gid.ctypes.data, bound.priority.ctypes.data, bound.start_ns.ctypes.data,
                                       bound.flags.ctypes.data))
    total = _lib().bsw_walk(C.byref(nd), C.byref(pd), C.byref(b), idx.ctypes.data if n else None, n,
                            last.ctypes.data if n else None, int(gang), node.ctypes.data, nv.ctypes.data,
                            cand.ctypes.data, outcome.ctypes.data, vict.ctypes.data, evby.ctypes.data)
    off = np.zeros(n + 1, np.uint32)
    off[1:] = np.cumsum(nv)
    assert total == off[-1]
    return WalkResult(node, nv, cand, off, vict[:total].copy(), outcome, evby[:V].copy())


def warm():
    """Compiles and loads the restatement (first use compiles it with gcc)."""
    _lib()
