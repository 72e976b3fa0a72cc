"""TEST INFRASTRUCTURE — the CPU restatement of bs_preempt and bs_preempt_walk under the PodFitsHostPorts filter
(include/bsched.h bs_upload_bound_host_ports).

tests/preempt_host_ports_ref.c keeps each node's used ports as a set of (ip, protocol, port) tuples with HostPortInfo's
Add / Remove / CheckConflict, on top of tests/preempt_pdb_ref.c's single-pod preemption and tests/preempt_walk_ref.c's
walk, whose helpers it includes.  It is compiled on first use into a library of its own in tests/native.py's build
directory, the way tests/preempt_walk_ref.py builds its file.

The filter's columns come as host_ports_ref.random_columns gives them: cols = ((entries [K, 3], used [N]), want [P]);
bound_ports [V] uint64 holds bit k when bound row v holds entry k.
"""
from __future__ import annotations

import ctypes as C
import functools
import os
import subprocess

import numpy as np

import native
from oracle import oracle
from preempt_ref import PreemptResult, _Bound
from preempt_walk_ref import WalkResult, units_last

_HERE = os.path.dirname(os.path.abspath(__file__))


class _Dict(C.Structure):
    _fields_ = [("n_entries", C.c_uint32), ("ip", C.c_void_p), ("protocol", C.c_void_p), ("port", C.c_void_p)]


@functools.cache
def _lib():
    so = oracle.build()
    out = os.path.join(native._out_dir().name, "libbs_preempt_host_ports_ref.so")
    subprocess.check_call(["gcc", "-O2", "-std=c11", "-fPIC", "-Wall", "-Wextra", "-fopenmp", "-shared", "-o", out,
                           os.path.join(_HERE, "preempt_host_ports_ref.c"), "-I" + _HERE,
                           "-I" + os.path.join(os.path.dirname(_HERE), "oracle"), so,
                           "-Wl,-rpath," + os.path.dirname(so), "-lm"])
    oracle.lib()   # the oracle library first, so that its symbols resolve
    lib = C.CDLL(out)
    common = [C.POINTER(oracle._Nodes), C.POINTER(oracle._Pods), C.POINTER(_Bound), C.POINTER(_Dict), C.c_void_p,
              C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32]
    lib.bshp_preempt.restype = None
    lib.bshp_preempt.argtypes = common + [C.c_void_p] * 4 + [C.c_uint32]
    lib.bshp_walk.restype = C.c_uint32
    lib.bshp_walk.argtypes = common + [C.c_void_p, C.c_int] + [C.c_void_p] * 6
    return lib


def warm():
    """Compiles and loads the restatement (first use compiles it with gcc)."""
    _lib()


def _args(snap, bound, cols, bound_ports):
    (entries, used), want = cols
    ent = np.asarray(entries, np.int64).reshape(-1, 3)
    keep = [np.ascontiguousarray(ent[:, 0], np.uint32), np.ascontiguousarray(ent[:, 1], np.uint32),
            np.ascontiguousarray(ent[:, 2], np.int32), np.ascontiguousarray(used, np.uint64),
            np.ascontiguousarray(np.zeros(max(bound.n, 1), np.uint64) if bound_ports is None else
                                 np.append(np.asarray(bound_ports, np.uint64), np.uint64(0))),
            np.ascontiguousarray(np.append(np.asarray(want, np.uint64), np.uint64(0)))]
    d = _Dict(len(ent), *(k.ctypes.data for k in keep[:3]))
    nd, pd = oracle._nodes(snap.nodes, getattr(snap, "aff_bits", None)), oracle._pods(snap.pods)
    b = _Bound(bound.n, bound.lanes, *(bound.node.ctypes.data, bound.req.ctypes.data, bound.req_present.ctypes.data,
                                       bound.gid.ctypes.data, bound.priority.ctypes.data, bound.start_ns.ctypes.data,
                                       bound.flags.ctypes.data))
    return (C.byref(nd), C.byref(pd), C.byref(b), C.byref(d), keep[3].ctypes.data, keep[4].ctypes.data,
            keep[5].ctypes.data), (keep, nd, pd, b, d)


def preempt(snap, bound, cols, bound_ports, pods=None) -> PreemptResult:
    """bs_preempt's outputs under the filter for the pod indices `pods` (all pods when None)."""
    idx = np.ascontiguousarray(np.arange(snap.pods.n) if pods is None else pods, dtype=np.uint32)
    n = len(idx)
    counts = np.bincount(bound.node.astype(np.int64), minlength=snap.nodes.n) if bound.n else np.zeros(1, np.int64)
    vstride = max(1, int(counts.max()) if len(counts) else 1)
    node, nv, cand = np.zeros(n, np.int32), np.zeros(n, np.uint32), np.zeros(n, np.uint32)
    vict = np.zeros((max(n, 1), vstride), np.uint32)
    args, _keep = _args(snap, bound, cols, bound_ports)
    _lib().bshp_preempt(*args, idx.ctypes.data if n else None, n, node.ctypes.data, nv.ctypes.data, cand.ctypes.data,
                        vict.ctypes.data, vstride)
    off = np.zeros(n + 1, np.uint32)
    off[1:] = np.cumsum(nv)
    victims = np.concatenate([vict[i, :nv[i]] for i in range(n)]).astype(np.uint32) if n else np.zeros(0, np.uint32)
    return PreemptResult(node, nv, cand, off, victims)


def walk(snap, bound, cols, bound_ports, pods, gang=False) -> WalkResult:
    """bs_preempt_walk's outputs under the filter for `pods` in list order (the caller keeps the engine's list rules)."""
    idx = np.ascontiguousarray(pods, dtype=np.uint32)
    n, V = len(idx), bound.n
    node, nv, cand, outcome = (np.zeros(n, np.int32), np.zeros(n, np.uint32), np.zeros(n, np.uint32),
                               np.zeros(n, np.uint32))
    vict = np.zeros(max(V, 1), np.uint32)
    evby = np.zeros(max(V, 1), np.int32)
    last = units_last(snap, idx, gang)
    args, _keep = _args(snap, bound, cols, bound_ports)
    total = _lib().bshp_walk(*args, idx.ctypes.data if n else None, n, last.ctypes.data if n else None, int(gang),
                             node.ctypes.data, nv.ctypes.data, cand.ctypes.data, outcome.ctypes.data,
                             vict.ctypes.data, evby.ctypes.data)
    off = np.zeros(n + 1, np.uint32)
    off[1:] = np.cumsum(nv)
    assert total == off[-1]
    return WalkResult(node, nv, cand, off, vict[:total].copy(), outcome, evby[:V].copy())


def random_bound_ports(snap, bound, used, seed: int, p_hold: float = 0.5) -> np.ndarray:
    """[V] uint64: each bound row holds a random subset of its node's used entries (each entry with p_hold)."""
    rng = np.random.default_rng(seed)
    used = np.asarray(used, np.uint64)
    out = np.zeros(bound.n, np.uint64)
    for v in range(bound.n):
        u = int(used[int(bound.node[v])])
        m = 0
        while u:
            bit = u & -u
            if rng.random() < p_hold:
                m |= bit
            u ^= bit
        out[v] = np.uint64(m)
    return out
