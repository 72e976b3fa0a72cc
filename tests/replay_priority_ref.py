"""TEST INFRASTRUCTURE — the CPU restatement of bs_replay_priority (include/bsched.h).

tests/replay_priority_ref.c restates the oracle's pod-at-a-time walk over the oracle's public helpers with the node
choice as a hook, and the scoring chooser over tests/priority_ref.c's scorer.  Both files are compiled with
-ffp-contract=off on first use into tests/native.py's library of the C restatements.
"""
from __future__ import annotations

import ctypes as C
import functools

import numpy as np

import native
from oracle import oracle

DEFAULT_WEIGHTS = (1, 0, 1)


@functools.cache
def _lib():
    lib = native.ref_lib()
    P = C.c_void_p
    lib.bsr_replay_priority.argtypes = [C.POINTER(oracle._Nodes), C.POINTER(oracle._Pods),
                                        C.POINTER(oracle._Groups), P, C.c_uint32, P, P, P, P, P,
                                        C.c_uint32, C.c_uint32, C.c_uint32]
    lib.bsr_replay_choose.argtypes = [C.POINTER(oracle._Nodes), C.POINTER(oracle._Pods),
                                      C.POINTER(oracle._Groups), P, C.c_uint32, P, P, P, P, P, P]
    lib.bsr_first_fit.restype = C.c_int32
    lib.bsr_priority_choose.restype = C.c_int32
    return lib


def _walk(snap, queue, call):
    s = snap.copy()
    nt, pt, gt = s.nodes, s.pods, s.groups
    q = np.ascontiguousarray(np.arange(pt.n) if queue is None else queue, dtype=np.uint32)
    pf, node, ready = np.zeros(len(q), np.uint8), np.zeros(len(q), np.int32), np.zeros(len(q), np.uint8)
    if pt.aff_class is not None and gt.rep_aff is None:
        gt.rep_aff = np.full(gt.n, oracle.AFF_NONE, np.uint32)   # the walk records the first pod's class here
    nd, pd, gr = oracle._nodes(nt, getattr(s, "aff_bits", None)), oracle._pods(pt), oracle._groups(gt)
    call(C.byref(nd), C.byref(pd), C.byref(gr), q.ctypes.data, len(q), pf.ctypes.data, node.ctypes.data,
         ready.ctypes.data)
    return pf, node, ready, s


def replay_priority(snap, node_nz, pod_nz, queue=None, weights=DEFAULT_WEIGHTS):
    """bs_replay_priority on COPIES of the tables: (prefilter, node, ready, snap_after, node_nonzero_after [2, N])."""
    live = np.array(node_nz, dtype=np.int64).reshape(2, snap.nodes.n)
    pod_nz = np.ascontiguousarray(pod_nz, dtype=np.int64).reshape(2, snap.pods.n)
    f = _lib().bsr_replay_priority
    pf, node, ready, s = _walk(snap, queue, lambda *a: f(*a, live.ctypes.data, pod_nz.ctypes.data, *weights))
    return pf, node, ready, s, live


def replay_first_fit(snap, queue=None):
    """The hooked walk with bso_replay's first-fit chooser: (prefilter, node, ready, snap_after)."""
    lib = _lib()
    first_fit = C.cast(lib.bsr_first_fit, C.c_void_p)
    return _walk(snap, queue, lambda *a: lib.bsr_replay_choose(*a, first_fit, None, None))
