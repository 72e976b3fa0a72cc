"""TEST INFRASTRUCTURE — the CPU restatement of the MatchInterPodAffinity filter (include/bsched.h
bs_set_interpod_filter) on the packed columns.

tests/interpod_filter_ref.c loops over the bound pods for each (pod, node), with no presence tables, and returns the
step that failed.  It is compiled on first use into a library of its own in tests/native.py's temporary directory.
verdicts() gives the verdict matrix, expected() the engine's outputs restated: the oracle's fit ANDed with the filter,
and the companion reason rows.
"""
from __future__ import annotations

import ctypes as C
import functools
import os
import subprocess

import numpy as np

import native

PASS, FAIL_E, FAIL_A, FAIL_N = range(4)
_HERE = os.path.dirname(os.path.abspath(__file__))


class _Ipf(C.Structure):
    _fields_ = [("n_nodes", C.c_uint32), ("topo", C.c_void_p), ("term_key", C.c_void_p), ("n_bound", C.c_uint32),
                ("bound_node", C.c_void_p), ("bound_class", C.c_void_p), ("b_off", C.c_void_p), ("b_term", C.c_void_p),
                ("b_own", C.c_void_p), ("b_match", C.c_void_p), ("pod_class", C.c_void_p), ("p_off", C.c_void_p),
                ("p_term", C.c_void_p), ("p_role", C.c_void_p), ("p_self", C.c_void_p)]


@functools.cache
def _lib():
    out = os.path.join(native._out_dir().name, "libbs_interpod_filter_ref.so")
    subprocess.check_call(["gcc", "-O2", "-std=c11", "-fPIC", "-Wall", "-Wextra", "-shared", "-o", out,
                           os.path.join(_HERE, "interpod_filter_ref.c")])
    lib = C.CDLL(out)
    lib.bsr_ipf_verdict.restype = C.c_int
    lib.bsr_ipf_verdict.argtypes = [C.POINTER(_Ipf), C.c_uint32, C.c_uint32]
    lib.bsr_ipf_matrix.restype = None
    lib.bsr_ipf_matrix.argtypes = [C.POINTER(_Ipf), C.c_void_p, C.c_uint32, C.c_void_p]
    return lib


def verdicts(columns, n_nodes: int, pods=None) -> np.ndarray:
    """[n, N] uint8: PASS / FAIL_E / FAIL_A / FAIL_N of every pod (or the pod indices `pods`) on every node, for
    columns = (node, pods) as snapshot.node_interpod_filter returns them."""
    (nv, topo, tkey, bnode, bcls, (boff, bterm, bown, bmatch)), (pcls, (poff, pterm, prole, pself)) = columns
    u32 = lambda a: np.ascontiguousarray(a, dtype=np.uint32).reshape(-1)
    u8 = lambda a: np.ascontiguousarray(a, dtype=np.uint8).reshape(-1)
    keep = [u32(topo) if len(nv) else np.zeros(1, np.uint32), u32(tkey), u32(bnode), u32(bcls), u32(boff), u32(bterm),
            np.ascontiguousarray(bown, dtype=np.int32).reshape(-1), u8(bmatch), u32(pcls), u32(poff), u32(pterm),
            u8(prole), u8(pself)]
    a = [x.ctypes.data for x in keep]
    q = _Ipf(n_nodes, a[0], a[1], len(keep[2]), *a[2:])
    idx = np.arange(len(keep[8]), dtype=np.uint32) if pods is None else np.ascontiguousarray(pods, dtype=np.uint32)
    out = np.zeros((len(idx), n_nodes), np.uint8)
    if len(idx) and n_nodes:
        _lib().bsr_ipf_matrix(C.byref(q), idx.ctypes.data, len(idx), out.ctypes.data)
    return out


def companion_rows(v: np.ndarray, lane_ok: np.ndarray) -> np.ndarray:
    """[n, 3] uint32 (E, A, N): per pod, the nodes that pass every other check (lane_ok [n, N] bool: the guards,
    checkFit and every lane) and then fail the filter at each step."""
    return np.stack([((v == s) & lane_ok).sum(1) for s in (FAIL_E, FAIL_A, FAIL_N)], 1).astype(np.uint32)
