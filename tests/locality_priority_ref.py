"""TEST INFRASTRUCTURE — the CPU restatement of the ImageLocality and NodePreferAvoidPods priorities
(include/bsched.h bs_set_locality_weights) in the priority lists and in bs_replay_priority.

tests/locality_priority_ref.c counts each name's nodes, scales its size in binary64, sums a pod's class over the names
a node reports and adds both terms to tests/ratio_priority_ref.c's resource score (and, in the lists, to
tests/node_priority_ref.c's TaintToleration and NodeAffinity terms).  It is compiled on first use, with the flags of
tests/native.py's library of the C restatements, into a library of its own in that library's temporary directory,
linked against it, against tests/node_priority_ref.py's library and against the oracle.
"""
from __future__ import annotations

import ctypes as C
import functools
import os
import subprocess

import numpy as np

import native
import node_priority_ref as npr
import ratio_priority_ref as rref
from oracle import oracle

DEFAULT_WEIGHTS = (1, 0, 1)
NO_RATIO = npr.NO_RATIO


class _Loc(C.Structure):
    _fields_ = [("image_size", C.c_void_p), ("image_bits", C.c_void_p), ("avoid_mask", C.c_void_p),
                ("n_images", C.c_uint32), ("image_class", C.c_void_p), ("class_offset", C.c_void_p),
                ("class_images", C.c_void_p), ("avoid_bit", C.c_void_p), ("scaled", C.c_void_p),
                ("w_img", C.c_uint32), ("w_avoid", C.c_uint32)]


_HERE = os.path.dirname(os.path.abspath(__file__))


@functools.cache
def _lib():
    ref = native.ref_lib()
    pref = npr._lib()   # loaded first: the node-priority scorer resolves from it
    so = oracle.build()
    out = os.path.join(os.path.dirname(ref._name), "libbs_locality_priority_ref.so")
    subprocess.check_call(["gcc", "-O2", "-std=c11", "-fPIC", "-Wall", "-Wextra", "-ffp-contract=off", "-shared", "-o",
                           out, os.path.join(_HERE, "locality_priority_ref.c"),
                           "-I" + os.path.join(os.path.dirname(_HERE), "oracle"), ref._name, pref._name, so,
                           "-Wl,-rpath," + os.path.dirname(ref._name) + ":" + os.path.dirname(so)])
    lib = C.CDLL(out)
    P, Q = C.c_void_p, C.POINTER(_Loc)
    lib.bsr_image_scaled.restype = C.c_int64
    lib.bsr_image_scaled.argtypes = [C.c_int64, C.c_uint32, C.c_uint32]
    lib.bsr_image_locality.restype = C.c_int64
    lib.bsr_image_locality.argtypes = [C.c_int64]
    lib.bsr_image_spread.restype = None
    lib.bsr_image_spread.argtypes = [Q, C.c_uint32, P]
    lib.bsr_il.restype = C.c_int64
    lib.bsr_il.argtypes = [Q, C.POINTER(oracle._Nodes), C.c_uint32, C.c_uint32]
    lib.bsr_npa.restype = C.c_int64
    lib.bsr_npa.argtypes = [Q, C.c_uint32, C.c_uint32]
    lib.bsr_locality_rows.restype = None
    lib.bsr_locality_rows.argtypes = [Q, C.POINTER(npr._Pref), C.POINTER(rref._Setting), C.POINTER(oracle._Nodes),
                                      C.POINTER(oracle._Pods), P, P, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                      C.c_uint32, P, P]
    lib.bsr_replay_locality.argtypes = [C.POINTER(oracle._Nodes), C.POINTER(oracle._Pods), C.POINTER(oracle._Groups),
                                        P, C.c_uint32, P, P, P, P, P, C.c_uint32, C.c_uint32, C.c_uint32,
                                        C.POINTER(rref._Setting), Q]
    return lib


def image_scaled(size, num_nodes, total_nodes) -> int:
    return int(_lib().bsr_image_scaled(size, num_nodes, total_nodes))


def image_locality(total) -> int:
    return int(_lib().bsr_image_locality(total))


class Columns:
    """The C struct over numpy copies of (node, pods) = ((image_size, image_bits, avoid_mask), (image_class,
    class_offset, class_images, avoid_bit)) with weights lw = (ImageLocality, NodePreferAvoidPods); keeps the arrays
    alive and fills scaled[] once."""

    def __init__(self, loc, n_nodes, lw):
        (size, bits, avoid), (cls, off, ids, abit) = loc
        self.arrays = [np.ascontiguousarray(size, dtype=np.int64),
                       np.ascontiguousarray(bits, dtype=np.uint32).reshape(len(size), (n_nodes + 31) // 32),
                       np.ascontiguousarray(avoid, dtype=np.uint64), np.ascontiguousarray(cls, dtype=np.uint32),
                       np.ascontiguousarray(off, dtype=np.uint32), np.ascontiguousarray(ids, dtype=np.uint32),
                       np.ascontiguousarray(abit, dtype=np.uint8)]
        self.scaled = np.zeros(max(len(size), 1), np.int64)
        a = self.arrays
        self.q = _Loc(a[0].ctypes.data, a[1].ctypes.data, a[2].ctypes.data, len(size), a[3].ctypes.data,
                      a[4].ctypes.data, a[5].ctypes.data, a[6].ctypes.data, self.scaled.ctypes.data, *lw)
        _lib().bsr_image_spread(C.byref(self.q), n_nodes, self.scaled.ctypes.data)


def scaled(loc, n_nodes):
    """scaled[i] of every name of the node side."""
    return Columns(loc, n_nodes, (1, 1)).scaled[:len(loc[0][0])].copy()


def il_matrix(snap, loc, pods=None):
    """[n, N] int64: IL of every pod (or the pod indices `pods`) on every node."""
    cols = Columns(loc, snap.nodes.n, (1, 1))
    nd = oracle._nodes(snap.nodes, getattr(snap, "aff_bits", None))
    idx = np.arange(snap.pods.n) if pods is None else np.asarray(pods, np.int64)
    f = _lib().bsr_il
    return np.array([[f(C.byref(cols.q), C.byref(nd), int(p), n) for n in range(snap.nodes.n)] for p in idx],
                    np.int64).reshape(len(idx), snap.nodes.n)


def npa_matrix(snap, loc):
    """[P, N] int64: NPA of every pod on every node."""
    cols = Columns(loc, snap.nodes.n, (1, 1))
    f = _lib().bsr_npa
    return np.array([[f(C.byref(cols.q), p, n) for n in range(snap.nodes.n)] for p in range(snap.pods.n)],
                    np.int64).reshape(snap.pods.n, snap.nodes.n)


def priority_rows(snap, node_nz, pod_nz, K, loc, lw, ratio=NO_RATIO, weights=DEFAULT_WEIGHTS, prefs=None, pw=(0, 0),
                  pods=None):
    """(nodes [n, K] int32, scores [n, K] int64) under the resource weights, the ratio setting, the node priorities
    (prefs = node_priority_ref's columns, pw their weights; None: off) and the locality priorities: loc = (node, pods)
    as snapshot.node_locality returns them, lw = (ImageLocality, NodePreferAvoidPods) weights."""
    nt, pt = snap.nodes, snap.pods
    idx = np.arange(pt.n) if pods is None else np.asarray(pods, np.int64)
    nodes = np.zeros((len(idx), K), np.int32)
    scores = np.zeros((len(idx), K), np.int64)
    node_nz = np.ascontiguousarray(node_nz, dtype=np.int64).reshape(2, nt.n)
    pod_nz = np.ascontiguousarray(pod_nz, dtype=np.int64).reshape(2, pt.n)
    cols = Columns(loc, nt.n, lw)
    pq = None
    if prefs is not None and any(pw):
        pcols = npr._columns(prefs, nt.n)
        pq = C.byref(npr._Pref(*(c.ctypes.data for c in pcols), *pw))
    lanes = list(ratio[2]) + [0] * (nt.lanes - len(ratio[2]))
    s = rref.setting(ratio[0], ratio[1], lanes, *ratio[3:])
    nd, pd = oracle._nodes(nt, getattr(snap, "aff_bits", None)), oracle._pods(pt)
    f = _lib().bsr_locality_rows
    for k, p in enumerate(idx):
        f(C.byref(cols.q), pq, C.byref(s), C.byref(nd), C.byref(pd), node_nz.ctypes.data, pod_nz.ctypes.data, int(p), K,
          *weights, nodes[k].ctypes.data, scores[k].ctypes.data)
    return nodes, scores


def replay_locality(snap, node_nz, pod_nz, loc, lw, ratio=NO_RATIO, queue=None, weights=DEFAULT_WEIGHTS):
    """bs_replay_priority with the locality terms on COPIES of the tables: (prefilter, node, ready, snap_after,
    node_nonzero_after [2, N])."""
    import replay_priority_ref as rpr
    live = np.array(node_nz, dtype=np.int64).reshape(2, snap.nodes.n)
    pod_nz = np.ascontiguousarray(pod_nz, dtype=np.int64).reshape(2, snap.pods.n)
    cols = Columns(loc, snap.nodes.n, lw)
    lanes = list(ratio[2]) + [0] * (snap.nodes.lanes - len(ratio[2]))
    s = rref.setting(ratio[0], ratio[1], lanes, *ratio[3:])
    f = _lib().bsr_replay_locality
    pf, node, ready, after = rpr._walk(snap, queue, lambda *a: f(*a, live.ctypes.data, pod_nz.ctypes.data, *weights,
                                                                   C.byref(s), C.byref(cols.q)))
    return pf, node, ready, after, live
