"""TEST INFRASTRUCTURE — the CPU restatement of the TaintToleration and preferred NodeAffinity priorities
(include/bsched.h bs_set_node_priority_weights) in the priority lists.

tests/node_priority_ref.c takes each pod's maxima over its fit set from the oracle's bso_fit_eval, normalizes both raw
counts and adds them to tests/ratio_priority_ref.c's resource score.  It is compiled on first use, with the flags of
tests/native.py's library of the C restatements, into a library of its own in that library's temporary directory,
linked against it (for bsr_ratio_total) and against the oracle.
"""
from __future__ import annotations

import ctypes as C
import functools
import os
import subprocess

import numpy as np

import native
import ratio_priority_ref as rref
from oracle import oracle

DEFAULT_WEIGHTS = (1, 0, 1)
NO_RATIO = (0, rref.DEFAULT_SHAPE, [0] * 4)


class _Pref(C.Structure):
    _fields_ = [("prefer_taints", C.c_void_p), ("pref_weights", C.c_void_p), ("prefer_tol", C.c_void_p),
                ("pref_class", C.c_void_p), ("w_taint", C.c_uint32), ("w_naff", C.c_uint32)]


_HERE = os.path.dirname(os.path.abspath(__file__))


@functools.cache
def _lib():
    ref = native.ref_lib()   # loaded first: bsr_ratio_total resolves from it
    so = oracle.build()
    out = os.path.join(os.path.dirname(ref._name), "libbs_node_priority_ref.so")
    subprocess.check_call(["gcc", "-O2", "-std=c11", "-fPIC", "-Wall", "-Wextra", "-ffp-contract=off", "-shared", "-o",
                           out, os.path.join(_HERE, "node_priority_ref.c"),
                           "-I" + os.path.join(os.path.dirname(_HERE), "oracle"), ref._name, so,
                           "-Wl,-rpath," + os.path.dirname(ref._name) + ":" + os.path.dirname(so)])
    lib = C.CDLL(out)
    P, Q = C.c_void_p, C.POINTER(_Pref)
    lib.bsr_node_priority_rows.restype = None
    lib.bsr_node_priority_rows.argtypes = [Q, C.POINTER(rref._Setting), C.POINTER(oracle._Nodes),
                                           C.POINTER(oracle._Pods), P, P, C.c_uint32, C.c_uint32, C.c_uint32,
                                           C.c_uint32, C.c_uint32, P, P]
    lib.bsr_node_pref_maxima.restype = None
    lib.bsr_node_pref_maxima.argtypes = [Q, C.POINTER(oracle._Nodes), C.POINTER(oracle._Pods), C.c_uint32, P, P]
    lib.bsr_normalize.restype = C.c_int64
    lib.bsr_normalize.argtypes = [C.c_int64, C.c_int64, C.c_int]
    return lib


def _columns(prefs, n_nodes):
    taints, table, tol, cls = prefs
    taints = np.ascontiguousarray(taints, dtype=np.uint64)
    table = np.ascontiguousarray(table, dtype=np.int32)
    table = table.reshape(len(table) if table.ndim == 2 else -1, n_nodes)   # [C, 0] for an empty node table
    tol = np.ascontiguousarray(tol, dtype=np.uint64)
    cls = np.ascontiguousarray(cls, dtype=np.uint32)
    return taints, table, tol, cls


def normalize(raw, mx, reverse) -> int:
    return int(_lib().bsr_normalize(raw, mx, 1 if reverse else 0))


def maxima(snap, prefs, pods=None):
    """[n, 2] int64: (Mt, Ma) of every pod (or the pod indices `pods`) over its fit set."""
    nt, pt = snap.nodes, snap.pods
    cols = _columns(prefs, nt.n)
    q = _Pref(*(c.ctypes.data for c in cols), 1, 1)
    nd, pd = oracle._nodes(nt, getattr(snap, "aff_bits", None)), oracle._pods(pt)
    idx = np.arange(pt.n) if pods is None else np.asarray(pods, np.int64)
    out = np.zeros((len(idx), 2), np.int64)
    mt, ma = C.c_int64(), C.c_int64()
    for k, p in enumerate(idx):
        _lib().bsr_node_pref_maxima(C.byref(q), C.byref(nd), C.byref(pd), int(p), C.addressof(mt), C.addressof(ma))
        out[k] = (mt.value, ma.value)
    return out


def priority_rows(snap, node_nz, pod_nz, K, prefs, pref_weights, ratio=NO_RATIO, weights=DEFAULT_WEIGHTS, pods=None):
    """(nodes [n, K] int32, scores [n, K] int64) under the resource weights, the ratio setting (weight, shape,
    lane_weights[, absent_weight]) and the node priorities: prefs = (prefer_taints [N], pref_weights [C, N],
    prefer_tol [P], pref_class [P]), pref_weights = (TaintToleration, NodeAffinity) weights."""
    nt, pt = snap.nodes, snap.pods
    idx = np.arange(pt.n) if pods is None else np.asarray(pods, np.int64)
    nodes = np.zeros((len(idx), K), np.int32)
    scores = np.zeros((len(idx), K), np.int64)
    node_nz = np.ascontiguousarray(node_nz, dtype=np.int64).reshape(2, nt.n)
    pod_nz = np.ascontiguousarray(pod_nz, dtype=np.int64).reshape(2, pt.n)
    cols = _columns(prefs, nt.n)
    q = _Pref(*(c.ctypes.data for c in cols), *pref_weights)
    lw = list(ratio[2]) + [0] * (nt.lanes - len(ratio[2]))
    s = rref.setting(ratio[0], ratio[1], lw, *ratio[3:])
    nd, pd = oracle._nodes(nt, getattr(snap, "aff_bits", None)), oracle._pods(pt)
    f = _lib().bsr_node_priority_rows
    for k, p in enumerate(idx):
        f(C.byref(q), C.byref(s), C.byref(nd), C.byref(pd), node_nz.ctypes.data, pod_nz.ctypes.data, int(p), K,
          *weights, nodes[k].ctypes.data, scores[k].ctypes.data)
    return nodes, scores
