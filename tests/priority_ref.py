"""TEST INFRASTRUCTURE — the CPU restatement of the priority lists (include/bsched.h BS_OUT_PRIORITY).

tests/priority_ref.c takes each pod's fit set from the oracle's bso_fit_eval and restates the three resource scorers in
C.  It is compiled with -ffp-contract=off into a temporary directory on first use, because the tree may be read-only,
and linked against oracle/libbs_oracle.so.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from oracle import oracle

_HERE = os.path.dirname(os.path.abspath(__file__))
_ORACLE_DIR = os.path.join(os.path.dirname(_HERE), "oracle")
_lib_cache = None

DEFAULT_WEIGHTS = (1, 0, 1)


def _lib():
    global _lib_cache
    if _lib_cache is None:
        so = oracle.build()
        out = os.path.join(tempfile.mkdtemp(prefix="priority_ref_"), "libpriority_ref.so")
        subprocess.check_call(["gcc", "-O2", "-std=c11", "-fPIC", "-Wall", "-Wextra", "-ffp-contract=off", "-shared",
                               "-o", out, os.path.join(_HERE, "priority_ref.c"), "-I" + _ORACLE_DIR, so, "-lm",
                               "-Wl,-rpath," + os.path.dirname(so)])
        oracle.lib()   # the oracle library first, so that its symbols resolve
        lib = C.CDLL(out)
        lib.bsr_priority_rows.restype = None
        lib.bsr_priority_rows.argtypes = [C.POINTER(oracle._Nodes), C.POINTER(oracle._Pods), C.c_void_p, C.c_void_p,
                                          C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p,
                                          C.c_void_p]
        lib.bsr_priority_score.restype = C.c_int64
        lib.bsr_priority_score.argtypes = [C.c_int64] * 4 + [C.c_uint32] * 3
        _lib_cache = lib
    return _lib_cache


def score(r_cpu, c_cpu, r_mem, c_mem, weights=DEFAULT_WEIGHTS) -> int:
    """The weighted score of one (requested, capacity) pair per resource."""
    return int(_lib().bsr_priority_score(r_cpu, c_cpu, r_mem, c_mem, *weights))


def priority_rows(snap, node_nz, pod_nz, K, weights=DEFAULT_WEIGHTS, pods=None):
    """(nodes [n, K] int32, scores [n, K] int64) for every pod, or only the pod indices `pods`."""
    nt, pt = snap.nodes, snap.pods
    idx = np.arange(pt.n) if pods is None else np.asarray(pods, np.int64)
    nodes = np.zeros((len(idx), K), np.int32)
    scores = np.zeros((len(idx), K), np.int64)
    node_nz = np.ascontiguousarray(node_nz, dtype=np.int64).reshape(2, nt.n)
    pod_nz = np.ascontiguousarray(pod_nz, dtype=np.int64).reshape(2, pt.n)
    nd, pd = oracle._nodes(nt, getattr(snap, "aff_bits", None)), oracle._pods(pt)
    f = _lib().bsr_priority_rows
    for k, p in enumerate(idx):
        f(C.byref(nd), C.byref(pd), node_nz.ctypes.data, pod_nz.ctypes.data, int(p), K, *weights,
          nodes[k].ctypes.data, scores[k].ctypes.data)
    return nodes, scores
