"""TEST INFRASTRUCTURE — the CPU restatement of the RequestedToCapacityRatio priority (include/bsched.h
bs_set_ratio_priority) in the priority lists and in bs_replay_priority.

tests/ratio_priority_ref.c restates the ratio term from the broken-line definition and adds it to tests/priority_ref.c's
scorer; its list builder takes the fit set from the oracle's bso_fit_eval, and its chooser / assume hooks drive
tests/replay_priority_ref.c's walk.  The three files are compiled with -ffp-contract=off on first use into
tests/native.py's library of the C restatements.
"""
from __future__ import annotations

import ctypes as C
import functools

import numpy as np

import native
from oracle import oracle

DEFAULT_WEIGHTS = (1, 0, 1)
DEFAULT_SHAPE = ((0, 100), (100, 0))   # v1.17's default {(0, 10), (100, 0)} in node-score units
BIN_PACK = ((0, 0), (100, 100))


class _Setting(C.Structure):
    _fields_ = [("weight", C.c_uint32), ("n_points", C.c_uint32), ("utilization", C.c_int64 * 101),
                ("score", C.c_int64 * 101), ("n_lanes", C.c_uint32), ("lane_weight", C.c_uint32 * 16),
                ("absent_weight", C.c_uint32)]


def setting(weight, shape, lane_weights, absent_weight=0):
    """The C setting struct of (weight, [(utilization, score), ...], [weight per lane], absent_weight)."""
    s = _Setting()
    s.weight, s.n_points, s.n_lanes, s.absent_weight = weight, len(shape), len(lane_weights), absent_weight
    for i, (u, v) in enumerate(shape):
        s.utilization[i], s.score[i] = u, v
    for d, w in enumerate(lane_weights):
        s.lane_weight[d] = w
    return s


@functools.cache
def _lib():
    lib = native.ref_lib()
    P, S = C.c_void_p, C.POINTER(_Setting)
    lib.bsr_ratio_shape.restype = C.c_int64
    lib.bsr_ratio_shape.argtypes = [S, C.c_int64]
    lib.bsr_ratio_util.restype = C.c_int64
    lib.bsr_ratio_util.argtypes = [C.c_int64, C.c_int64]
    lib.bsr_ratio_of.restype = C.c_int64
    lib.bsr_ratio_of.argtypes = [S, P, P]
    lib.bsr_ratio_rows.restype = None
    lib.bsr_ratio_rows.argtypes = [S, C.POINTER(oracle._Nodes), C.POINTER(oracle._Pods), P, P, C.c_uint32,
                                   C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, P, P]
    lib.bsr_replay_ratio.argtypes = [C.POINTER(oracle._Nodes), C.POINTER(oracle._Pods), C.POINTER(oracle._Groups),
                                     P, C.c_uint32, P, P, P, P, P, C.c_uint32, C.c_uint32, C.c_uint32, S]
    return lib


def shape_at(shape, p) -> int:
    return int(_lib().bsr_ratio_shape(C.byref(setting(0, shape, [0] * 4)), p))


def utilization(r, c) -> int:
    return int(_lib().bsr_ratio_util(r, c))


def ratio_of(shape, lane_weights, r, c, absent_weight=0) -> int:
    """Ratio of per-lane requested r and capacity c (missing keys as 0)."""
    rr = np.ascontiguousarray(r, dtype=np.int64)
    cc = np.ascontiguousarray(c, dtype=np.int64)
    return int(_lib().bsr_ratio_of(C.byref(setting(0, shape, lane_weights, absent_weight)), rr.ctypes.data,
                                   cc.ctypes.data))


def priority_rows(snap, node_nz, pod_nz, K, ratio, weights=DEFAULT_WEIGHTS, pods=None):
    """(nodes [n, K] int32, scores [n, K] int64) under weights + the ratio setting (weight, shape, lane_weights[,
    absent_weight]), for every pod or only the pod indices `pods`."""
    nt, pt = snap.nodes, snap.pods
    idx = np.arange(pt.n) if pods is None else np.asarray(pods, np.int64)
    nodes = np.zeros((len(idx), K), np.int32)
    scores = np.zeros((len(idx), K), np.int64)
    node_nz = np.ascontiguousarray(node_nz, dtype=np.int64).reshape(2, nt.n)
    pod_nz = np.ascontiguousarray(pod_nz, dtype=np.int64).reshape(2, pt.n)
    nd, pd = oracle._nodes(nt, getattr(snap, "aff_bits", None)), oracle._pods(pt)
    s = setting(*ratio)
    f = _lib().bsr_ratio_rows
    for k, p in enumerate(idx):
        f(C.byref(s), C.byref(nd), C.byref(pd), node_nz.ctypes.data, pod_nz.ctypes.data, int(p), K, *weights,
          nodes[k].ctypes.data, scores[k].ctypes.data)
    return nodes, scores


def replay_ratio(snap, node_nz, pod_nz, ratio, queue=None, weights=DEFAULT_WEIGHTS):
    """bs_replay_priority with the ratio setting on COPIES of the tables: (prefilter, node, ready, snap_after,
    node_nonzero_after [2, N])."""
    import replay_priority_ref as rpr
    live = np.array(node_nz, dtype=np.int64).reshape(2, snap.nodes.n)
    pod_nz = np.ascontiguousarray(pod_nz, dtype=np.int64).reshape(2, snap.pods.n)
    s = setting(*ratio)
    f = _lib().bsr_replay_ratio
    pf, node, ready, after = rpr._walk(snap, queue, lambda *a: f(*a, live.ctypes.data, pod_nz.ctypes.data, *weights,
                                                                   C.byref(s)))
    return pf, node, ready, after, live
