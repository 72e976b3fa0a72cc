"""CPU: the two restatements of the priority lists (BS_OUT_PRIORITY) agree — tests/priority_ref.c (fit set from the
oracle's bso_fit_eval) and tests/pyref_priority.py (pure Python) — on random snapshots and on hand-built cases covering
every branch of the three scorers; the C ABI's flag, list-length rule and the packer's non-zero columns."""
import json
import os
import re
import subprocess

import numpy as np
import pytest

import native
import priority_ref
import pyref_priority
from randsnap import random_snapshot

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WEIGHTS = [(1, 0, 1), (0, 1, 0), (3, 2, 5), (0, 0, 0), (1, 1, 1)]
M56 = 1 << 56
I64_MIN = -(1 << 63)


def _as_lists(nodes, scores):
    return [[(int(n), int(s)) for n, s in zip(rn, rs)] for rn, rs in zip(nodes, scores)]


# -- the scorers, branch by branch ---------------------------------------------------------------------------------
# (r_cpu, c_cpu, r_mem, c_mem): requested (non-zero, pod included) and allocatable of cpu and memory
CASES = {
    "capacity 0": (5, 0, 10, 100),                   # cpu scores 0, its fraction is 1.0: Balanced 0
    "both capacities 0": (0, 0, 0, 0),
    "requested > capacity": (101, 100, 50, 100),     # cpu scores 0, fraction >= 1
    "requested == capacity": (100, 100, 0, 100),     # cpu least 0 / most 100, fraction == 1
    "fraction >= 1 on memory": (10, 100, 200, 100),
    "negative allocatable": (10, -100, 30, 100),     # a fraction <= 0
    "44 not 45": (10, 1000, 560, 1000),
    "exact halves": (50, 100, 50, 100),
    "near 2^56": (M56 - 1, M56, M56 // 3, M56),      # (2^56 - 1) / 2^56 rounds to 1.0 in binary64
    "saturating Balanced": (2 * M56, -1, 0, M56),    # (1 - 2^57) * 100 is below -2^63
}


def _expected_parts(r_cpu, c_cpu, r_mem, c_mem):
    return (pyref_priority._trunc_div(pyref_priority.least_requested(r_cpu, c_cpu) +
                                      pyref_priority.least_requested(r_mem, c_mem), 2),
            pyref_priority._trunc_div(pyref_priority.most_requested(r_cpu, c_cpu) +
                                      pyref_priority.most_requested(r_mem, c_mem), 2),
            pyref_priority.balanced(r_cpu, c_cpu, r_mem, c_mem))


@pytest.mark.parametrize("name", sorted(CASES))
def test_scorer_branches(name):
    args = CASES[name]
    least, most, bal = _expected_parts(*args)
    # each part alone through the C restatement
    assert priority_ref.score(*args, weights=(1, 0, 0)) == least
    assert priority_ref.score(*args, weights=(0, 1, 0)) == most
    assert priority_ref.score(*args, weights=(0, 0, 1)) == bal
    for w in WEIGHTS:
        assert priority_ref.score(*args, weights=w) == pyref_priority.score(*args, weights=w), w


def test_hand_computed_values():
    assert _expected_parts(10, 1000, 560, 1000) == (71, 28, 44)     # float64 gives 44.99999999999999, not 45
    assert (1 - abs(10 / 1000 - 560 / 1000)) * 100.0 == 44.99999999999999
    assert _expected_parts(5, 0, 10, 100) == (45, 5, 0)
    assert _expected_parts(101, 100, 50, 100) == (25, 25, 0)
    assert _expected_parts(100, 100, 0, 100) == (50, 50, 0)
    assert _expected_parts(50, 100, 50, 100) == (50, 50, 100)
    # a negative capacity: cpu scores 0, its fraction is -0.1, so Balanced = (1 - 0.4) * 100 truncated, below 100
    least, most, bal = _expected_parts(10, -100, 30, 100)
    assert (least, most) == (35, 15) and 0 < bal <= 60
    assert _expected_parts(M56 - 1, M56, M56 // 3, M56) == (33, 66, 0)
    assert _expected_parts(2 * M56, -1, 0, M56) == (50, 0, I64_MIN)
    assert _expected_parts(M56, -1, 0, M56)[2] == int((1 - 2.0 ** 56) * 100.0)   # still inside int64
    # weights wrap in int64: 3 * 50 + 5 * INT64_MIN
    want = ((3 * 50 + 5 * I64_MIN) + (1 << 63)) % (1 << 64) - (1 << 63)
    assert priority_ref.score(2 * M56, -1, 0, M56, weights=(3, 0, 5)) == want
    assert pyref_priority.score(2 * M56, -1, 0, M56, (3, 0, 5)) == want


def test_float64_disagrees_with_exact_often():
    """Pairs of fractions k/100 where binary64 and rational arithmetic disagree on Balanced."""
    n = 0
    for a in range(100):
        for b in range(100):
            exact = 100 - abs(a - b)
            if pyref_priority.balanced(a, 100, b, 100) != exact:
                n += 1
                assert priority_ref.score(a, 100, b, 100, weights=(0, 0, 1)) == exact - 1
    assert n > 100


def test_random_pairs_agree():
    rng = np.random.default_rng(7)
    caps = np.concatenate([rng.integers(-1000, 1 << 20, 300), rng.integers(0, M56, 300), [0, 1, -1, M56, -M56]])
    for _ in range(3000):
        c_cpu, c_mem = (int(x) for x in rng.choice(caps, 2))
        r_cpu = int(rng.integers(0, max(abs(c_cpu), 1) * 2 + 1)) if rng.random() < 0.8 else int(rng.integers(0, M56))
        r_mem = int(rng.integers(0, max(abs(c_mem), 1) * 2 + 1)) if rng.random() < 0.8 else int(rng.integers(0, M56))
        r_cpu, r_mem = min(r_cpu, 2 * M56), min(r_mem, 2 * M56)
        w = WEIGHTS[int(rng.integers(len(WEIGHTS)))]
        assert priority_ref.score(r_cpu, c_cpu, r_mem, c_mem, w) == pyref_priority.score(r_cpu, c_cpu, r_mem, c_mem, w)


# -- whole lists ----------------------------------------------------------------------------------------------------
def random_case(seed, L, P=40, N=70, aff=0):
    import importlib
    S = importlib.import_module("batch-scheduler_b200.snapshot")
    snap = random_snapshot(seed, P=P, N=N, G=8, L=L, aff=aff)
    node_nz, pod_nz = S.nonzero_requests(snap, seed)
    return snap, node_nz, pod_nz


@pytest.mark.parametrize("L", [4, 5, 9, 16])
@pytest.mark.parametrize("wi", range(len(WEIGHTS)))
def test_restatements_agree_on_random_snapshots(oracle, L, wi):
    snap, node_nz, pod_nz = random_case(1000 + 17 * L + wi, L, aff=3 if L % 2 else 0)
    w = WEIGHTS[wi]
    for K in (1, 7, 32):
        got = _as_lists(*priority_ref.priority_rows(snap, node_nz, pod_nz, K, w))
        assert got == pyref_priority.priority_rows(snap, node_nz, pod_nz, K, w), K


def tie_snapshot():
    """60 identical nodes but three, so that almost every score ties; the fit set is every node but the skipped ones."""
    import importlib
    S = importlib.import_module("batch-scheduler_b200.snapshot")
    N, P, L = 60, 6, 4
    nt = S.NodeTable.empty(N, L)
    nt.alloc[0], nt.alloc[1], nt.alloc[2], nt.alloc[3] = 4000, 8 << 30, 100 << 30, 110
    nt.requested[0], nt.requested[1] = 1000, 2 << 30
    nt.alloc[0, 10] = 8000                     # a better LeastAllocated node in the middle
    nt.alloc[0, 40] = nt.requested[0, 40] = 0  # cpu capacity 0: only the pod without a cpu request fits it
    nt.flags[5] = S.NODE_UNSCHEDULABLE
    pt = S.PodTable.empty(P, L)
    pt.req[0] = [100, 500, 4000, 0, 100, 100]
    pt.req[1] = [1 << 20, 1 << 30, 1 << 30, 0, 1 << 20, 1 << 20]
    gt = S.GroupTable.empty(2, L)
    gt.min_member[:] = 1
    snap = S.Snapshot(nt, pt, gt, "ties")
    node_nz = np.stack([nt.requested[0], nt.requested[1]]).astype(np.int64)
    pod_nz = np.stack([np.where(pt.req[0] == 0, 100, pt.req[0]), np.where(pt.req[1] == 0, 200 << 20, pt.req[1])])
    return snap, node_nz, pod_nz.astype(np.int64)


@pytest.mark.parametrize("w", WEIGHTS)
def test_ties_across_many_nodes(oracle, w):
    snap, node_nz, pod_nz = tie_snapshot()
    for K in (1, 7, 32):
        nodes, scores = priority_ref.priority_rows(snap, node_nz, pod_nz, K, w)
        assert _as_lists(nodes, scores) == pyref_priority.priority_rows(snap, node_nz, pod_nz, K, w)
        for rn, rs in zip(nodes, scores):
            real = rn[rn >= 0]
            assert 5 not in real.tolist()
            # score descending, then index ascending
            keys = [(-int(s), int(n)) for n, s in zip(rn, rs) if n >= 0]
            assert keys == sorted(keys)
    nodes, _ = priority_ref.priority_rows(snap, node_nz, pod_nz, 7, (1, 0, 1))
    assert nodes[0].tolist() == [0, 1, 2, 3, 4, 6, 7]   # equal scores by index; the roomier node 10 is less balanced
    node40 = pyref_priority.Node(snap.nodes, 40)
    assert pyref_priority.fits(node40, snap.pods, 3, 40, None, 4) and not pyref_priority.fits(node40, snap.pods, 0, 40, None, 4)


# -- the C ABI --------------------------------------------------------------------------------------------------------
def test_flag_agrees_across_header_and_capi(pkg):
    hdr = open(os.path.join(ROOT, "include", "bsched.h")).read()
    m = re.search(r"#define BS_OUT_PRIORITY (0x[0-9a-fA-F]+)u", hdr)
    assert m and int(m.group(1), 16) == pkg.capi.OUT_PRIORITY == 0x20
    m = re.search(r"#define BS_NONZERO_MAX \(1ll << (\d+)\)", hdr)
    assert m and 1 << int(m.group(1)) == pkg.capi.NONZERO_MAX == 1 << 56
    for f in (pkg.capi.OUT_FIT_BITMAP, pkg.capi.OUT_SCORE, pkg.capi.OUT_FILTER, pkg.capi.OUT_TOPK, pkg.capi.OUT_REASONS):
        assert not f & pkg.capi.OUT_PRIORITY
    assert pkg.capi.KERNEL_NAMES == ["node_left", "find_max", "class_prefix", "prefilter", "gang_fit", "sort", "filter",
                                     "peer", "replay"]


def _create(pkg, flags, k):
    import ctypes as C
    lib = pkg.capi.load()
    cfg = pkg.capi.Config(0, 5, flags, k)
    h = C.c_void_p()
    rc = lib.bs_create(C.byref(cfg), C.byref(h))
    if rc == 0:
        lib.bs_destroy(h)
    return rc


def test_create_list_length_rule(pkg):
    c = pkg.capi
    P = c.OUT_PRIORITY
    for k in (0, 33, 1000):
        assert _create(pkg, P, k) == c.BS_E_INVAL
        assert _create(pkg, P | c.OUT_TOPK, k) == c.BS_E_INVAL
    others = [c.OUT_FIT_BITMAP, c.OUT_SCORE, c.OUT_FILTER, c.OUT_TOPK, c.OUT_REASONS]
    for mask in range(1 << len(others)):
        flags = P | sum(f for i, f in enumerate(others) if mask >> i & 1)
        want_ok = not (flags & c.OUT_TOPK and flags & c.OUT_SCORE)
        for k in (1, 16, 32):
            rc = _create(pkg, flags, k)
            assert (rc in (c.BS_OK, c.BS_E_NODEVICE)) if want_ok else rc == c.BS_E_INVAL, (flags, k, rc)
    # the rule without the new flag keeps its answers
    assert _create(pkg, c.OUT_FIT_BITMAP, 1) == c.BS_E_INVAL
    assert _create(pkg, c.OUT_TOPK, 0) == c.BS_E_INVAL
    assert _create(pkg, c.OUT_TOPK | c.OUT_SCORE, 4) == c.BS_E_INVAL


def test_engine_rejects_unequal_list_lengths(pkg):
    with pytest.raises(ValueError):
        pkg.Engine(5, topk=4, priority_k=8)


# -- the packer -------------------------------------------------------------------------------------------------------
def test_packer_nonzero_columns():
    o = json.loads(subprocess.check_output([native.cpp_program("plugin_priority_test"), "pack"], text=True))
    d_cpu, d_mem = 100, 200 << 20
    # pods: no containers; one container without requests; explicit zeros; set values; cpu only; two containers;
    # limits only (Requests, not Limits, count)
    assert o["pod_cpu"] == [0, d_cpu, 0, 1500, 250, 250 + d_cpu, d_cpu]
    assert o["pod_mem"] == [0, d_mem, 0, 3 << 30, d_mem, (1 << 30) + d_mem, d_mem]
    # nodes: no pods; the pods of rows 1-3; a nil NodeInfo
    assert o["node_cpu"] == [0, d_cpu + 1500, 250 + 250 + d_cpu, 0]
    assert o["node_mem"] == [0, d_mem + (3 << 30), d_mem + (1 << 30) + d_mem, 0]
    assert o["bad"] == 1
