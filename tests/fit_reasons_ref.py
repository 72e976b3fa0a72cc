"""TEST INFRASTRUCTURE — the CPU restatement of the reason rows (include/bsched.h BS_OUT_REASONS).

tests/fit_reasons_ref.c builds each row from the oracle's own helpers (bso_check_fit, bso_single_node_resource,
bso_pod_require).  It is compiled on first use into tests/native.py's library of the C restatements.
"""
from __future__ import annotations

import ctypes as C
import functools

import numpy as np

import native
from oracle import oracle


@functools.cache
def _lib():
    f = native.ref_lib().bsr_fit_reasons
    f.restype = None
    f.argtypes = [C.POINTER(oracle._Nodes), C.POINTER(oracle._Pods), C.c_uint32, C.POINTER(C.c_uint32)]
    return f


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
