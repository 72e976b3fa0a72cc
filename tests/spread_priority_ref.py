"""TEST INFRASTRUCTURE — the CPU restatement of the SelectorSpread priority (include/bsched.h bs_set_spread_weight) in
the priority lists.

tests/spread_priority_ref.c reduces each pod's counts over its fit set (the oracle's bso_fit_eval) as
CalculateSpreadPriorityReduce does, blends the node and zone scores in binary64 and adds the result to
tests/ratio_priority_ref.c's resource score, and, when given, to tests/node_priority_ref.c's TaintToleration and
NodeAffinity terms and tests/locality_priority_ref.c's locality terms.  It is compiled on first use, with the flags of
tests/native.py's library of the C restatements, into a library of its own in that library's temporary directory,
linked against it, against the node-priority and locality libraries and against the oracle.
"""
from __future__ import annotations

import ctypes as C
import functools
import os
import subprocess

import numpy as np

import locality_priority_ref as lpr
import native
import node_priority_ref as npr
import ratio_priority_ref as rref
from oracle import oracle

DEFAULT_WEIGHTS = (1, 0, 1)
NO_RATIO = npr.NO_RATIO


class _Spread(C.Structure):
    _fields_ = [("zone", C.c_void_p), ("counts", C.c_void_p), ("spread_class", C.c_void_p), ("w_spread", C.c_uint32)]


_HERE = os.path.dirname(os.path.abspath(__file__))


@functools.cache
def _lib():
    ref = native.ref_lib()
    pref = npr._lib()   # loaded first: the node-priority and locality terms resolve from them
    loc = lpr._lib()
    so = oracle.build()
    out = os.path.join(os.path.dirname(ref._name), "libbs_spread_priority_ref.so")
    subprocess.check_call(["gcc", "-O2", "-std=c11", "-fPIC", "-Wall", "-Wextra", "-ffp-contract=off", "-shared", "-o",
                           out, os.path.join(_HERE, "spread_priority_ref.c"),
                           "-I" + os.path.join(os.path.dirname(_HERE), "oracle"), ref._name, pref._name, loc._name, so,
                           "-Wl,-rpath," + os.path.dirname(ref._name) + ":" + os.path.dirname(so)])
    lib = C.CDLL(out)
    P, Q = C.c_void_p, C.POINTER(_Spread)
    lib.bsr_spread_score.restype = C.c_int64
    lib.bsr_spread_score.argtypes = [C.c_int64, C.c_int64, C.c_int, C.c_int64, C.c_int64]
    lib.bsr_spread_reduce.restype = None
    lib.bsr_spread_reduce.argtypes = [Q, C.POINTER(oracle._Nodes), C.POINTER(oracle._Pods), C.c_uint32, P]
    lib.bsr_spread_rows.restype = None
    lib.bsr_spread_rows.argtypes = [Q, C.POINTER(npr._Pref), P, C.POINTER(rref._Setting), C.POINTER(oracle._Nodes),
                                    C.POINTER(oracle._Pods), P, P, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                    C.c_uint32, P, P]
    return lib


def spread_score(max_node, count, zoned, max_zone, zone_count) -> int:
    """SS of one node from its count, the pod's largest count, and (zoned) its zone's sum and the largest zone sum."""
    return int(_lib().bsr_spread_score(max_node, count, 1 if zoned else 0, max_zone, zone_count))


class Columns:
    """The C struct over numpy copies of spread = ((zone [N], counts [C, N]), spread_class [P]) with weight w."""

    def __init__(self, spread, n_nodes, w):
        (zone, counts), cls = spread
        self.arrays = [np.ascontiguousarray(zone, dtype=np.uint8).reshape(n_nodes),
                       np.ascontiguousarray(counts, dtype=np.int32).reshape(np.shape(counts)[0] if np.ndim(counts) == 2 else -1,
                                                                          n_nodes),
                       np.ascontiguousarray(cls, dtype=np.uint32)]
        self.q = _Spread(*(a.ctypes.data for a in self.arrays), w)


def ss_matrix(snap, spread, pods=None):
    """[n, N] int64: SS of every pod (or the pod indices `pods`) on every node; -1 where the pod does not fit."""
    nt, pt = snap.nodes, snap.pods
    cols = Columns(spread, nt.n, 1)
    nd, pd = oracle._nodes(nt, getattr(snap, "aff_bits", None)), oracle._pods(pt)
    idx = np.arange(pt.n) if pods is None else np.asarray(pods, np.int64)
    out = np.full((len(idx), nt.n), -1, np.int64)
    for k, p in enumerate(idx):
        _lib().bsr_spread_reduce(C.byref(cols.q), C.byref(nd), C.byref(pd), int(p), out[k].ctypes.data)
    return out


def priority_rows(snap, node_nz, pod_nz, K, spread, w_spread, ratio=NO_RATIO, weights=DEFAULT_WEIGHTS, prefs=None,
                  pw=(0, 0), loc=None, lw=(0, 0), pods=None):
    """(nodes [n, K] int32, scores [n, K] int64) under the resource weights, the ratio setting, the node priorities
    (prefs = node_priority_ref's columns, pw their weights), the locality priorities (loc = snapshot.node_locality's
    columns, lw their weights) and SelectorSpread: spread = snapshot.node_spread's columns, w_spread its weight.  A
    priority whose columns are None or whose weights are all 0 is off."""
    nt, pt = snap.nodes, snap.pods
    idx = np.arange(pt.n) if pods is None else np.asarray(pods, np.int64)
    nodes = np.zeros((len(idx), K), np.int32)
    scores = np.zeros((len(idx), K), np.int64)
    node_nz = np.ascontiguousarray(node_nz, dtype=np.int64).reshape(2, nt.n)
    pod_nz = np.ascontiguousarray(pod_nz, dtype=np.int64).reshape(2, pt.n)
    cols = Columns(spread, nt.n, w_spread)
    pq = None
    if prefs is not None and any(pw):
        pcols = npr._columns(prefs, nt.n)
        pq = C.byref(npr._Pref(*(c.ctypes.data for c in pcols), *pw))
    lq, lcols = None, None
    if loc is not None and any(lw):
        lcols = lpr.Columns(loc, nt.n, lw)
        lq = C.addressof(lcols.q)
    lanes = list(ratio[2]) + [0] * (nt.lanes - len(ratio[2]))
    s = rref.setting(ratio[0], ratio[1], lanes, *ratio[3:])
    nd, pd = oracle._nodes(nt, getattr(snap, "aff_bits", None)), oracle._pods(pt)
    f = _lib().bsr_spread_rows
    for k, p in enumerate(idx):
        f(C.byref(cols.q), pq, lq, C.byref(s), C.byref(nd), C.byref(pd), node_nz.ctypes.data, pod_nz.ctypes.data,
          int(p), K, *weights, nodes[k].ctypes.data, scores[k].ctypes.data)
    return nodes, scores
