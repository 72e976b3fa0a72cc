"""CPU: the reason rows of the round (include/bsched.h BS_OUT_REASONS) on two CPU restatements — tests/fit_reasons_ref.c,
built on the C oracle's helpers, and tests/pyref_reasons.py — and the FailedScheduling text of bs_format_fit_error,
which needs no device.  The GPU rows are compared with the C restatement in tests/test_gpu_fit_reasons.py."""
import itertools
import os
import re

import numpy as np
import pytest

import fit_reasons_ref
import lane_cases
import pyref_reasons
import randsnap
import reason_cases

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
R_SEEDS = [(seed, L, scale, aff) for seed, (L, scale, aff) in
           enumerate(itertools.product((4, 5, 6, 9, 12, 16), ("normal", "big"), (0, 7)))]


def _invariant(oracle, snap, rows):
    """A node counts in no bin <=> the pod fits it: per pod, nodes with a bin = N - feasible_count."""
    r = oracle.round(snap, want_bitmap=True)
    N = snap.nodes.n
    fit = np.unpackbits(r.fit_bitmap.view(np.uint8), axis=1, bitorder="little")[:, :N].astype(bool)
    assert np.array_equal(fit.sum(axis=1), r.feasible_count)
    assert np.all(rows[:, :2].sum(axis=1) <= N)   # a guarded node counts in one guard bin
    hit = (rows > 0).any(axis=1)
    assert np.array_equal(hit, r.feasible_count < N)
    return r


@pytest.mark.parametrize("seed,L,scale,aff", R_SEEDS)
def test_oracle_agrees_with_pyref_random(oracle, seed, L, scale, aff):
    snap = randsnap.random_snapshot(seed, P=60, N=75, G=12, L=L, value_scale=scale, aff=aff)
    rows = fit_reasons_ref.fit_reasons(snap)
    assert rows.shape == (60, 4 + L) and rows.dtype == np.uint32
    np.testing.assert_array_equal(rows, pyref_reasons.fit_reasons(snap))
    _invariant(oracle, snap, rows)


@pytest.mark.parametrize("L,d,case", lane_cases.combos())
def test_oracle_agrees_with_pyref_lane_cases(oracle, L, d, case):
    snap = lane_cases.small_snapshot(L, case, d, seed=3)
    rows = fit_reasons_ref.fit_reasons(snap)
    np.testing.assert_array_equal(rows, pyref_reasons.fit_reasons(snap))
    _invariant(oracle, snap, rows)
    assert rows[:, 4 + d].any(), "the deciding lane rejects some pod somewhere"


def test_invariant_nodes_with_a_bin_are_the_unfit_ones(oracle):
    """Per (pod, node): the node has a bin in the oracle's row of a one-node snapshot <=> the fit bit is clear."""
    snap = randsnap.random_snapshot(5, P=30, N=40, G=6, L=7, aff=4)
    full = oracle.round(snap, want_bitmap=True)
    N = snap.nodes.n
    fit = np.unpackbits(full.fit_bitmap.view(np.uint8), axis=1, bitorder="little")[:, :N].astype(bool)
    for n in range(N):
        one = snap.copy()
        nt = one.nodes
        for f in nt.__dataclass_fields__:
            a = getattr(nt, f)
            setattr(nt, f, np.ascontiguousarray(a[..., n:n + 1]))
        bit = (snap.aff_bits[:, n // 32] >> np.uint32(n % 32)) & np.uint32(1)
        one.aff_bits = bit.reshape(-1, 1).astype(np.uint32)
        rows = fit_reasons_ref.fit_reasons(one)
        np.testing.assert_array_equal((rows > 0).any(axis=1), ~fit[:, n])


def test_hand_built_table(oracle):
    snap = reason_cases.snapshot()
    want = reason_cases.expected()
    np.testing.assert_array_equal(want, [[3, 4, 4, 2, 2, 1, 1, 2, 4, 0], [3, 4, 0, 3, 0, 0, 0, 0, 0, 0]])
    np.testing.assert_array_equal(fit_reasons_ref.fit_reasons(snap), want)
    np.testing.assert_array_equal(pyref_reasons.fit_reasons(snap), want)
    r = _invariant(oracle, snap, want)
    fits = [k for k, (_, b0, _) in enumerate(reason_cases.NODES) if not b0]
    assert r.feasible_count[0] == len(fits)
    np.testing.assert_array_equal(fit_reasons_ref.fit_reasons(snap, pods=[1]), want[1:])


# ---- bs_format_fit_error -------------------------------------------------------------------------------------------

def _fmt(pkg, row, L, N, names=None, buf_len=4096):
    from importlib import import_module
    return import_module("batch-scheduler_b200.engine").format_fit_error(row, L, N, names, buf_len)


def test_format_exact_strings(pkg):
    row = [1, 2, 3, 4, 5, 6, 7, 8, 9]
    assert _fmt(pkg, row, 5, 60, ["nvidia.com/gpu"]) == (
        "0/60 nodes are available: 1 node(s) were unschedulable, 2 node(s) were unavailable, "
        "3 node(s) didn't match node selector, 4 node(s) had taints that the pod didn't tolerate, "
        "5 Insufficient cpu, 6 Insufficient memory, 7 Insufficient ephemeral-storage, 8 Insufficient pods, "
        "9 Insufficient nvidia.com/gpu.")


def test_format_sorts_whole_strings(pkg):
    """Go's sort.Strings: "10 ..." sorts before "9 ...", and equal counts sort by their text."""
    row = [9, 0, 0, 10, 4120, 0, 0, 0, 3, 3]
    assert _fmt(pkg, row, 6, 10000, ["example.com/fpga", "nvidia.com/gpu"]) == (
        "0/10000 nodes are available: 10 node(s) had taints that the pod didn't tolerate, "
        "3 Insufficient example.com/fpga, 3 Insufficient nvidia.com/gpu, 4120 Insufficient cpu, "
        "9 node(s) were unschedulable.")


def test_format_omits_zero_bins_and_all_zero_row(pkg):
    assert _fmt(pkg, [0, 0, 7, 0, 0, 0, 0, 0], 4, 7) == "0/7 nodes are available: 7 node(s) didn't match node selector."
    assert _fmt(pkg, [0] * 8, 4, 0) == "0/0 nodes are available: ."


def test_format_null_scalar_names(pkg):
    row = [0] * 4 + [0] * 4 + [1, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 2]
    assert _fmt(pkg, row, 16, 3) == "0/3 nodes are available: 1 Insufficient lane4, 2 Insufficient lane15."
    # a name list with a gap (NULL entry) falls back per lane
    assert _fmt(pkg, [0] * 8 + [1, 1], 6, 3, ["a.io/x"]) == \
        "0/3 nodes are available: 1 Insufficient a.io/x, 1 Insufficient lane5."


def test_format_buffer_one_byte_too_small(pkg):
    row = [1, 0, 0, 0, 2, 0, 0, 0]
    msg = _fmt(pkg, row, 4, 3)
    assert msg == "0/3 nodes are available: 1 node(s) were unschedulable, 2 Insufficient cpu."
    assert _fmt(pkg, row, 4, 3, buf_len=len(msg) + 1) == msg
    with pytest.raises(pkg.capi.BsError) as ei:
        _fmt(pkg, row, 4, 3, buf_len=len(msg))
    assert ei.value.code == pkg.capi.BS_E_INVAL


def test_format_rejects_bad_lane_count(pkg):
    import ctypes as C
    lib = pkg.capi.load()
    row = np.zeros(20, np.uint32)
    buf = C.create_string_buffer(64)
    for L in (3, 17):
        assert lib.bs_format_fit_error(row.ctypes.data, L, 1, None, buf, 64) == pkg.capi.BS_E_INVAL


# ---- ABI ----------------------------------------------------------------------------------------------------------

def test_header_and_capi_constants_agree(pkg):
    hdr = open(os.path.join(ROOT, "include", "bsched.h")).read()
    capi = pkg.capi
    assert int(re.search(r"#define BS_OUT_REASONS (0x[0-9a-f]+)u", hdr).group(1), 16) == capi.OUT_REASONS == 0x10
    for name in ("UNSCHEDULABLE", "UNAVAILABLE", "SELECTOR", "TAINTS", "LANE0"):
        v = int(re.search(r"#define BS_REASON_%s (\d+)" % name, hdr).group(1))
        assert v == getattr(capi, "REASON_" + name), name
    assert int(re.search(r"BS_K_REASONS = (\d+)", hdr).group(1)) == capi.K_REASONS == 9
    assert int(re.search(r"BS_K_COUNT = (\d+)", hdr).group(1)) == capi.K_COUNT == 10
    assert len(capi.KERNEL_NAMES) == capi.K_REASONS   # the per-kernel dictionary keeps its keys
    assert int(re.search(r"#define BS_ABI_VERSION (\d+)", hdr).group(1)) == capi.load().bs_abi_version() == 8


def test_create_accepts_reasons_with_every_flag_combination(pkg):
    import ctypes as C
    import torch
    capi = pkg.capi
    lib = capi.load()
    want = capi.BS_OK if torch.cuda.is_available() else capi.BS_E_NODEVICE
    others = (capi.OUT_FIT_BITMAP, capi.OUT_SCORE, capi.OUT_FILTER, capi.OUT_TOPK)
    n = 0
    for k in range(len(others) + 1):
        for combo in itertools.combinations(others, k):
            flags = capi.OUT_REASONS | sum(combo)
            if (flags & capi.OUT_TOPK) and (flags & capi.OUT_SCORE):
                continue
            cfg = capi.Config(0, 6, flags, 4 if flags & capi.OUT_TOPK else 0)
            h = C.c_void_p()
            rc = lib.bs_create(C.byref(cfg), C.byref(h))
            assert rc == want, (flags, rc)
            if rc == capi.BS_OK:
                lib.bs_destroy(h)
            n += 1
    assert n == 12
