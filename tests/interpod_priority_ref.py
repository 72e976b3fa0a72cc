"""TEST INFRASTRUCTURE — the CPU restatement of the InterPodAffinity priority (include/bsched.h bs_set_interpod_weight)
in the priority lists.

tests/interpod_priority_ref.c computes each pod's raw score from the packed columns as upstream does (a topologyScore
per key and value over the bound pods, not the engine's term x value tables), reduces it over the pod's fit set (the
oracle's bso_fit_eval) and adds the result to tests/spread_priority_ref.c's score parts: the resource score and, when
given, the node, locality and spread terms.  It is compiled on first use, with the flags of tests/native.py's library
of the C restatements, into a library of its own in that library's temporary directory, linked against it, against
the node-priority, locality and spread libraries and against the oracle.
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
import spread_priority_ref as spr
from oracle import oracle

DEFAULT_WEIGHTS = (1, 0, 1)
NO_RATIO = npr.NO_RATIO


class _Ipa(C.Structure):
    _fields_ = [("n_keys", C.c_uint32), ("n_values", C.c_void_p), ("topo", C.c_void_p), ("n_terms", C.c_uint32),
                ("term_key", C.c_void_p), ("n_bound", C.c_uint32), ("bound_node", C.c_void_p), ("bound_class", C.c_void_p),
                ("b_off", C.c_void_p), ("b_term", C.c_void_p), ("b_own", C.c_void_p), ("b_match", C.c_void_p),
                ("pod_class", C.c_void_p), ("p_off", C.c_void_p), ("p_term", C.c_void_p), ("p_own", C.c_void_p),
                ("p_match", C.c_void_p), ("w_ipa", C.c_uint32)]


_HERE = os.path.dirname(os.path.abspath(__file__))


@functools.cache
def _lib():
    ref = native.ref_lib()
    pref = npr._lib()   # loaded first: the node-priority, locality and spread terms resolve from them
    loc = lpr._lib()
    spread = spr._lib()
    so = oracle.build()
    out = os.path.join(os.path.dirname(ref._name), "libbs_interpod_priority_ref.so")
    subprocess.check_call(["gcc", "-O2", "-std=c11", "-fPIC", "-Wall", "-Wextra", "-ffp-contract=off", "-shared", "-o",
                           out, os.path.join(_HERE, "interpod_priority_ref.c"),
                           "-I" + os.path.join(os.path.dirname(_HERE), "oracle"), ref._name, pref._name, loc._name,
                           spread._name, so, "-Wl,-rpath," + os.path.dirname(ref._name) + ":" + os.path.dirname(so)])
    lib = C.CDLL(out)
    P, Q = C.c_void_p, C.POINTER(_Ipa)
    lib.bsr_ipa_score.restype = C.c_int64
    lib.bsr_ipa_score.argtypes = [C.c_int64, C.c_int64, C.c_int64]
    lib.bsr_ipa_raw.restype = None
    lib.bsr_ipa_raw.argtypes = [Q, C.c_uint32, C.c_uint32, P]
    lib.bsr_ipa_reduce.restype = None
    lib.bsr_ipa_reduce.argtypes = [Q, C.POINTER(oracle._Nodes), C.POINTER(oracle._Pods), C.c_uint32, P]
    lib.bsr_interpod_rows.restype = None
    lib.bsr_interpod_rows.argtypes = [Q, P, C.POINTER(npr._Pref), P, C.POINTER(rref._Setting),
                                      C.POINTER(oracle._Nodes), C.POINTER(oracle._Pods), P, P, C.c_uint32, C.c_uint32,
                                      C.c_uint32, C.c_uint32, C.c_uint32, P, P]
    return lib


def ipa_score(raw, mn, mx) -> int:
    """IPA of one node from its raw score and the pod's extremes over its fit set (both started at 0)."""
    return int(_lib().bsr_ipa_score(raw, mn, mx))


class Columns:
    """The C struct over numpy copies of interpod = (node, pods) as snapshot.node_interpod returns them, weight w."""

    def __init__(self, interpod, n_nodes, w):
        (nv, topo, tkey, bnode, bcls, bcl), (pcls, pcl) = interpod
        u32 = lambda a: np.ascontiguousarray(a, dtype=np.uint32).reshape(-1)
        nv = u32(nv)
        cl = lambda c: [u32(c[0]), u32(c[1]), np.ascontiguousarray(c[2], dtype=np.int32),
                        np.ascontiguousarray(c[3], dtype=np.uint8)]
        self.arrays = [nv, u32(topo) if len(nv) else np.zeros(1, np.uint32), u32(tkey), u32(bnode), u32(bcls),
                       *cl(bcl), u32(pcls), *cl(pcl)]
        a = [x.ctypes.data for x in self.arrays]
        self.q = _Ipa(len(nv), a[0], a[1], len(self.arrays[2]), a[2], len(self.arrays[3]), *a[3:], w)


def raw_matrix(interpod, n_nodes, pods=None):
    """[n, N] int64: the raw score of every pod (or the pod indices `pods`) on every node."""
    N = n_nodes
    cols = Columns(interpod, N, 1)
    idx = np.arange(len(interpod[1][0])) if pods is None else np.asarray(pods, np.int64)
    out = np.zeros((len(idx), N), np.int64)
    for k, p in enumerate(idx):
        _lib().bsr_ipa_raw(C.byref(cols.q), N, int(p), out[k].ctypes.data)
    return out


def ipa_matrix(snap, interpod, pods=None):
    """[n, N] int64: IPA of every pod (or the pod indices `pods`) on every node; -1 where the pod does not fit."""
    nt, pt = snap.nodes, snap.pods
    cols = Columns(interpod, nt.n, 1)
    nd, pd = oracle._nodes(nt, getattr(snap, "aff_bits", None)), oracle._pods(pt)
    idx = np.arange(pt.n) if pods is None else np.asarray(pods, np.int64)
    out = np.full((len(idx), nt.n), -1, np.int64)
    for k, p in enumerate(idx):
        _lib().bsr_ipa_reduce(C.byref(cols.q), C.byref(nd), C.byref(pd), int(p), out[k].ctypes.data)
    return out


def priority_rows(snap, node_nz, pod_nz, K, interpod, w_ipa, ratio=NO_RATIO, weights=DEFAULT_WEIGHTS, prefs=None,
                  pw=(0, 0), loc=None, lw=(0, 0), spread=None, w_spread=0, pods=None):
    """(nodes [n, K] int32, scores [n, K] int64) under the resource weights, the ratio setting, the node priorities
    (prefs, pw), the locality priorities (loc, lw), SelectorSpread (spread = snapshot.node_spread's columns, w_spread)
    and InterPodAffinity: interpod = snapshot.node_interpod's columns, w_ipa its weight.  A priority whose columns are
    None or whose weights are all 0 is off."""
    nt, pt = snap.nodes, snap.pods
    idx = np.arange(pt.n) if pods is None else np.asarray(pods, np.int64)
    nodes = np.zeros((len(idx), K), np.int32)
    scores = np.zeros((len(idx), K), np.int64)
    node_nz = np.ascontiguousarray(node_nz, dtype=np.int64).reshape(2, nt.n)
    pod_nz = np.ascontiguousarray(pod_nz, dtype=np.int64).reshape(2, pt.n)
    cols = Columns(interpod, nt.n, w_ipa)
    pq = None
    if prefs is not None and any(pw):
        pcols = npr._columns(prefs, nt.n)
        pq = C.byref(npr._Pref(*(c.ctypes.data for c in pcols), *pw))
    lq, lcols = None, None
    if loc is not None and any(lw):
        lcols = lpr.Columns(loc, nt.n, lw)
        lq = C.addressof(lcols.q)
    sq, scols = None, None
    if spread is not None and w_spread:
        scols = spr.Columns(spread, nt.n, w_spread)
        sq = C.addressof(scols.q)
    lanes = list(ratio[2]) + [0] * (nt.lanes - len(ratio[2]))
    s = rref.setting(ratio[0], ratio[1], lanes, *ratio[3:])
    nd, pd = oracle._nodes(nt, getattr(snap, "aff_bits", None)), oracle._pods(pt)
    f = _lib().bsr_interpod_rows
    for k, p in enumerate(idx):
        f(C.byref(cols.q), sq, pq, lq, C.byref(s), C.byref(nd), C.byref(pd), node_nz.ctypes.data, pod_nz.ctypes.data,
          int(p), K, *weights, nodes[k].ctypes.data, scores[k].ctypes.data)
    return nodes, scores
