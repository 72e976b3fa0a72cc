"""TEST INFRASTRUCTURE — the CPU restatement of the PodFitsHostPorts filter (include/bsched.h bs_set_host_port_filter)
on the packed columns, and what a round with it on answers.

tests/host_ports_ref.c compares every wanted entry with every used entry of each (pod, node); it is compiled on first
use into a library of its own in tests/native.py's temporary directory.  passes() gives the pass matrix,
companion_rows() the ports companion of the reason rows, replay() the walks with the filter on (its hook pair around
the first-fit, priority and ratio choosers of bsr_replay_choose), and expected_round() every output of a round with the
filter on: interpod_filter_ref's construction (the oracle's round on a copy of the snapshot in which each pod's affinity row
is ANDed with the filter's pass bits), with the ports pass bits ANDed in as well.
"""
from __future__ import annotations

import ctypes as C
import functools
import os
import subprocess

import numpy as np

import fit_reasons_ref as frr
import interpod_filter_ref as fr
import native
from oracle import oracle

_HERE = os.path.dirname(os.path.abspath(__file__))
GUARD_FLAGS = 0x0F   # BS_NODE_NIL | BS_NODE_NO_NODE | BS_NODE_UNSCHEDULABLE | BS_NODE_TAINTS_ERR: bins 0 and 1


class _Dict(C.Structure):
    _fields_ = [("n_entries", C.c_uint32), ("ip", C.c_void_p), ("protocol", C.c_void_p), ("port", C.c_void_p)]


@functools.cache
def _lib():
    out = os.path.join(native._out_dir().name, "libbs_host_ports_ref.so")
    subprocess.check_call(["gcc", "-O2", "-std=c11", "-fPIC", "-Wall", "-Wextra", "-shared", "-o", out,
                           os.path.join(_HERE, "host_ports_ref.c"), "-I" + os.path.join(os.path.dirname(_HERE), "oracle"),
                           "-I" + _HERE])
    lib = C.CDLL(out)
    lib.bsr_hp_pass.restype = C.c_int
    lib.bsr_hp_pass.argtypes = [C.POINTER(_Dict), C.c_uint64, C.c_uint64]
    lib.bsr_hp_matrix.restype = None
    lib.bsr_hp_matrix.argtypes = [C.POINTER(_Dict), C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p]
    return lib


def _dict(entries):
    """(the C dictionary, the arrays it points at)."""
    ent = np.asarray(entries, np.int64).reshape(-1, 3)
    keep = [np.ascontiguousarray(ent[:, 0], np.uint32), np.ascontiguousarray(ent[:, 1], np.uint32),
            np.ascontiguousarray(ent[:, 2], np.int32)]
    return _Dict(len(ent), *(k.ctypes.data for k in keep)), keep


def passes(entries, used, want) -> np.ndarray:
    """[P, N] bool: pod p passes PodFitsHostPorts on node n, for the columns of Engine.upload_host_ports."""
    d, keep = _dict(entries)
    used = np.ascontiguousarray(used, np.uint64)
    want = np.ascontiguousarray(want, np.uint64)
    out = np.zeros((len(want), len(used)), np.uint8)
    if out.size:
        _lib().bsr_hp_matrix(C.byref(d), want.ctypes.data, len(want), used.ctypes.data, len(used), out.ctypes.data)
    return out.astype(bool)


class _Ctx(C.Structure):
    _fields_ = [("inner", C.c_void_p), ("inner_assumed", C.c_void_p), ("inner_ctx", C.c_void_p), ("dict", _Dict),
                ("live", C.c_void_p), ("want", C.c_void_p)]


class _PriorityCtx(C.Structure):   # bsr_priority_ctx; bsr_ratio_ctx adds the setting
    _fields_ = [("node_nz", C.c_void_p), ("pod_nz", C.c_void_p), ("w_least", C.c_uint32), ("w_most", C.c_uint32),
                ("w_balanced", C.c_uint32)]


class _RatioCtx(C.Structure):
    _fields_ = _PriorityCtx._fields_ + [("s", C.c_void_p)]


def replay(snap, cols, queue=None, nz=None, weights=(1, 0, 1), ratio=None):
    """The walk with the filter on, on COPIES of the tables: bso_replay's first fit (nz None), bs_replay_priority's
    chooser (nz = (node_nz, pod_nz)) or with the ratio term too (ratio as ratio_priority_ref.setting takes it).
    Returns (prefilter, node, ready, snap_after, live used masks [N], live non-zero column [2, N] or None)."""
    import ratio_priority_ref as rr
    import replay_priority_ref as rpr
    ref = rpr._lib()
    fn = lambda name: C.cast(getattr(ref, name), C.c_void_p).value
    (entries, used), want = cols
    d, keep = _dict(entries)
    live = np.array(used, dtype=np.uint64)
    want = np.ascontiguousarray(want, dtype=np.uint64)
    nz_live = None
    if nz is None:
        inner, inner_assumed, inner_ctx = fn("bsr_first_fit"), None, None
    else:
        nz_live = np.array(nz[0], dtype=np.int64).reshape(2, snap.nodes.n)
        pod_nz = np.ascontiguousarray(nz[1], dtype=np.int64).reshape(2, snap.pods.n)
        keep += [pod_nz]
        if ratio is None:
            ictx = _PriorityCtx(nz_live.ctypes.data, pod_nz.ctypes.data, *weights)
            inner, inner_assumed = fn("bsr_priority_choose"), fn("bsr_priority_assumed")
        else:
            rr._lib()
            setting = rr.setting(*ratio)
            keep.append(setting)
            ictx = _RatioCtx(nz_live.ctypes.data, pod_nz.ctypes.data, *weights, C.addressof(setting))
            inner, inner_assumed = fn("bsr_ratio_choose"), fn("bsr_ratio_assumed")
        keep.append(ictx)
        inner_ctx = C.addressof(ictx)
    ctx = _Ctx(inner, inner_assumed, inner_ctx, d, live.ctypes.data, want.ctypes.data)
    lib = _lib()
    choose, assumed = (C.cast(getattr(lib, n), C.c_void_p).value for n in ("bsr_hp_choose", "bsr_hp_assumed"))
    pf, node, ready, after = rpr._walk(snap, queue, lambda *a: ref.bsr_replay_choose(*a, choose, assumed,
                                                                                      C.addressof(ctx)))
    return pf, node, ready, after, live, nz_live


def companion_rows(snap, ok: np.ndarray) -> np.ndarray:
    """[P] uint32: per pod, the nodes past the guards (reason bins 0 and 1) that fail the filter."""
    guard = (snap.nodes.flags & GUARD_FLAGS) == 0
    return ((~ok) & guard[None, :]).sum(1).astype(np.uint32)


def random_columns(snap, seed: int, n_entries: int = 12, grouped: float = 0.3, node_bits: int = 2):
    """Generator columns: a dictionary of n_entries entries over a few ips, both protocols and a handful of ports,
    about `grouped` of the groups wanting one or two entries (every pod of a group the same), and each node using up
    to node_bits entries."""
    rng = np.random.default_rng(seed)
    seen, entries = set(), []
    while len(entries) < n_entries:
        e = (int(rng.choice([0, 0, 1, 2])), int(rng.integers(0, 2)), int(rng.choice([22, 1234, 29500, 8080, 6379])))
        if e not in seen:
            seen.add(e)
            entries.append(e)
    K = len(entries)
    used = np.zeros(snap.nodes.n, np.uint64)
    for n in range(snap.nodes.n):
        for _ in range(int(rng.integers(0, node_bits + 1))):
            used[n] |= np.uint64(1) << np.uint64(rng.integers(0, K))
    gwant = np.zeros(max(snap.groups.n, 1), np.uint64)
    for g in range(snap.groups.n):
        if rng.random() < grouped:
            for _ in range(int(rng.integers(1, 3))):
                gwant[g] |= np.uint64(1) << np.uint64(rng.integers(0, K))
    gid = snap.pods.gid
    ok = (gid >= 0) & (gid < snap.groups.n)
    want = np.where(ok, gwant[np.clip(gid, 0, max(snap.groups.n - 1, 0))], np.uint64(0)).astype(np.uint64)
    return (np.array(entries, np.int64), used), want


def expected_round(snap, ok, cfg, lists=None, ipf_v=None):
    """Every output of a round with the filter on (and, with ipf_v the inter-pod verdicts, the MatchInterPodAffinity
    filter too), as interpod_filter_ref.expected_round: fit-set outputs from the oracle on the filtered snapshot,
    PreFilter, the sort and BS_OUT_FILTER from the plain one, Permit readiness from both.  `host_port_rows` and, with
    ipf_v, `interpod_rows` are the companions: the latter counts the nodes that fit the plain round, pass the ports
    test and fail the inter-pod filter."""
    N = snap.nodes.n
    v = np.where(ok, fr.PASS, fr.FAIL_E).astype(np.uint8)
    if ipf_v is not None:
        v = np.where(ok, ipf_v, fr.FAIL_E).astype(np.uint8)
    fsnap = fr._filtered(snap, v)
    orc = oracle.round(fsnap, want_bitmap=True, want_score=True)
    plain = oracle.round(snap, want_bitmap=True, want_filter=cfg.get("filter", False))
    admit, bitmap = fr._admit(snap, plain.prefilter, orc.feasible_count, plain.admit)
    out = dict(prefilter=plain.prefilter, feasible_count=orc.feasible_count, best_node=orc.best_node,
               best_score=orc.best_score, admit=admit, admit_bitmap=bitmap, new_denied=plain.new_denied,
               order=plain.order, rank=plain.rank, max_group=plain.max_group, max_finished=plain.max_finished)
    if cfg.get("fit_bitmap"):
        out["fit_rows"] = orc.fit_bitmap
    if cfg.get("score"):
        out["score_rows"] = orc.score
    if cfg.get("filter"):
        out["filter_rows"], out["filter_code"] = plain.filter_bitmap, plain.filter_code
    if cfg.get("reasons"):
        out["reason_rows"] = frr.fit_reasons(snap)
        out["host_port_rows"] = companion_rows(snap, ok)
        if ipf_v is not None:
            fit = np.unpackbits(plain.fit_bitmap.view(np.uint8), axis=1, bitorder="little")[:, :N].astype(bool)
            out["interpod_rows"] = fr.companion_rows(ipf_v, fit & ok)
    if lists is not None:
        out.update(lists(fsnap, orc.score))
    return out, fsnap
