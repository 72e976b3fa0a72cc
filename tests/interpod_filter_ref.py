"""TEST INFRASTRUCTURE — the CPU restatement of the MatchInterPodAffinity filter (include/bsched.h
bs_set_interpod_filter) on the packed columns.

tests/interpod_filter_ref.c loops over the bound pods for each (pod, node), with no presence tables, and returns the
step that failed.  It is compiled on first use into a library of its own in tests/native.py's temporary directory.
verdicts() gives the verdict matrix, companion_rows() the companion reason rows, and expected_round() every output of
a round with the filter on: the oracle's round on a copy of the snapshot in which each pod gets an affinity row of its
own, its old row ANDed with the filter's pass bits, for the fit set, and the plain snapshot's round for the rest.
"""
from __future__ import annotations

import ctypes as C
import functools
import os
import subprocess

import copy

import numpy as np

import fit_reasons_ref as frr
import native
from oracle import oracle

PASS, FAIL_E, FAIL_A, FAIL_N = range(4)
AFF_NONE = 0xFFFFFFFF
ADMIT, WAIT, UNSCHEDULABLE = range(3)   # BS_ADMIT, BS_WAIT, BS_UNSCHEDULABLE
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


def pack_bits(b: np.ndarray) -> np.ndarray:
    """[P, N] bool -> [P, ceil(N/32)] uint32, bit n % 32 of word n / 32."""
    P, N = b.shape
    W = (N + 31) // 32
    pad = np.zeros((P, W * 32), np.uint64)
    pad[:, :N] = b
    return (pad.reshape(P, W, 32) << np.arange(32, dtype=np.uint64)).sum(2).astype(np.uint32)


def _filtered(snap, v):
    """The snapshot with pod p's affinity row ANDed with the filter's pass bits (v[p] == PASS); groups keep theirs."""
    P, N = v.shape
    W = (N + 31) // 32
    old = snap.aff_bits if snap.aff_bits is not None else np.zeros((0, W), np.uint32)
    ac = snap.pods.aff_class if snap.pods.aff_class is not None else np.full(P, AFF_NONE, np.uint32)
    base = np.where((ac == AFF_NONE)[:, None], np.uint32(0xFFFFFFFF), old[np.minimum(ac, max(len(old) - 1, 0))]
                    if len(old) else np.uint32(0xFFFFFFFF))
    rows = (base & pack_bits(v == PASS)).astype(np.uint32)
    out = copy.deepcopy(snap)
    out.aff_bits = np.ascontiguousarray(np.concatenate([old, rows]), dtype=np.uint32)
    out.pods.aff_class = (len(old) + np.arange(P)).astype(np.uint32)
    if out.groups.rep_aff is None:
        out.groups.rep_aff = np.full(out.groups.n, AFF_NONE, np.uint32)
    return out


def _admit(snap, prefilter, feasible, idle):
    """Permit readiness per group from each pod's PreFilter verdict and feasible count (gang_admit_kernel's rule);
    groups without a pod in the round keep `idle`."""
    gt, G = snap.groups, snap.groups.n
    gid = snap.pods.gid
    ok = (gid >= 0) & (gid < G)
    in_round = np.bincount(gid[ok], minlength=G)
    c = np.bincount(gid[ok], weights=((prefilter == 0) & (feasible > 0))[ok], minlength=G).astype(np.int64)
    need = (gt.min_member.astype(np.int64) - gt.scheduled) & 0xFFFFFFFF
    v = np.where(c == 0, UNSCHEDULABLE, np.where(gt.matched + c >= need, ADMIT, WAIT))
    admit = np.where(in_round > 0, v, idle).astype(np.uint8)
    bits = np.zeros(((G + 31) // 32) * 32, np.uint64)
    bits[:G] = admit == ADMIT
    return admit, (bits.reshape(-1, 32) << np.arange(32, dtype=np.uint64)).sum(1).astype(np.uint32)


def expected_round(snap, columns, cfg, lists=None):
    """Every output of a round with the filter on, for an engine built with cfg (fit_bitmap, score, filter, reasons):
    a dict keyed as Engine's accessors name them, and the filtered snapshot.  The fit-set outputs (feasible_count,
    best_node / best_score, the fit and score rows, and whatever lists(filtered snapshot, its [P, N] scores) returns:
    the top-K and priority lists) come from the oracle on the filtered snapshot; PreFilter, new_denied, the sort, the
    max_group / max_finished pair, the Filter matrix and its codes, and the reason rows from the plain one (the filter
    reaches neither PreFilter nor BS_OUT_FILTER); Permit readiness from both; the companion rows `interpod_rows` count
    the nodes that fit the plain round and fail the filter."""
    N = snap.nodes.n
    v = verdicts(columns, N)
    fsnap = _filtered(snap, v)
    orc = oracle.round(fsnap, want_bitmap=True, want_score=True)
    plain = oracle.round(snap, want_bitmap=True, want_filter=cfg.get("filter", False))
    a0, b0 = _admit(snap, plain.prefilter, plain.feasible_count, plain.admit)
    assert np.array_equal(a0, plain.admit) and np.array_equal(b0, plain.admit_bitmap)   # the rule restated holds
    admit, bitmap = _admit(snap, plain.prefilter, orc.feasible_count, plain.admit)
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
        fit = np.unpackbits(plain.fit_bitmap.view(np.uint8), axis=1, bitorder="little")[:, :N].astype(bool)
        out["interpod_rows"] = companion_rows(v, fit)
    if lists is not None:
        out.update(lists(fsnap, orc.score))
    return out, fsnap
