"""TEST INFRASTRUCTURE — the CPU restatement of the reason rows (include/bsched.h BS_OUT_REASONS).

tests/fit_reasons_ref.c builds each row from the oracle's own helpers (bso_check_fit, bso_single_node_resource,
bso_pod_require).  It is compiled into a temporary directory on first use, because the tree may be read-only, and
linked against oracle/libbs_oracle.so.
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
_fn = None


def _lib():
    global _fn
    if _fn is None:
        so = oracle.build()
        out = os.path.join(tempfile.mkdtemp(prefix="fit_reasons_ref_"), "libfit_reasons_ref.so")
        subprocess.check_call(["gcc", "-O2", "-std=c11", "-fPIC", "-Wall", "-Wextra", "-shared", "-o", out,
                               os.path.join(_HERE, "fit_reasons_ref.c"), "-I" + _ORACLE_DIR, so,
                               "-Wl,-rpath," + os.path.dirname(so)])
        oracle.lib()   # the oracle library first, so that its symbols resolve
        lib = C.CDLL(out)
        f = lib.bsr_fit_reasons
        f.restype = None
        f.argtypes = [C.POINTER(oracle._Nodes), C.POINTER(oracle._Pods), C.c_uint32, C.POINTER(C.c_uint32)]
        _fn = f
    return _fn


def fit_reasons(snap, pods=None) -> np.ndarray:
    """[P, 4 + L] uint32 reason rows, or only the rows of the pod indices `pods`."""
    nt, pt = snap.nodes, snap.pods
    idx = np.arange(pt.n) if pods is None else np.asarray(pods, np.int64)
    out = np.zeros((len(idx), 4 + nt.lanes), np.uint32)
    nd, pd = oracle._nodes(nt, getattr(snap, "aff_bits", None)), oracle._pods(pt)
    f = _lib()
    for k, p in enumerate(idx):
        f(C.byref(nd), C.byref(pd), int(p), out[k].ctypes.data_as(C.POINTER(C.c_uint32)))
    return out
