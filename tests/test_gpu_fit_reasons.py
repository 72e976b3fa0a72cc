"""GPU: the reason rows of a round (BS_OUT_REASONS) bit-exact against the CPU restatement tests/fit_reasons_ref.c
(built on the oracle's helpers), in every lane layout, at unaligned sizes, beside every other output mode, after row
updates, at cfg4 size, and through the C++ plugin's FitError."""
import json
import subprocess

import numpy as np
import pytest

import fit_reasons_ref
import lane_cases
import native
import reason_cases
from randsnap import S, random_snapshot


def _fit_matrix(words, N):
    return np.unpackbits(words.view(np.uint8), axis=1, bitorder="little")[:, :N].astype(bool)


def _run(pkg, snap, **kw):
    kw.setdefault("fit_bitmap", True)
    eng = pkg.Engine(snap.lanes, 0, reasons=True, **kw)
    try:
        eng.upload(snap)
        res = eng.evaluate()
        rows = eng.reason_rows()
        fit = eng.fit_rows() if kw["fit_bitmap"] else None
    finally:
        eng.close()
    return res, rows, fit


def _check(oracle, snap, res, rows, fit):
    N = snap.nodes.n
    assert rows.shape == (snap.pods.n, 4 + snap.lanes)
    np.testing.assert_array_equal(rows, fit_reasons_ref.fit_reasons(snap))
    # invariant: the nodes with a bin are exactly the unfit ones
    np.testing.assert_array_equal((rows > 0).any(axis=1), res.feasible_count < N)
    if fit is not None and N:
        m = _fit_matrix(fit, N)
        np.testing.assert_array_equal(m.sum(axis=1), res.feasible_count)
        assert np.all(rows[:, :2].sum(axis=1) <= (~m).sum(axis=1))


@pytest.mark.gpu
@pytest.mark.parametrize("L", range(4, 17))
@pytest.mark.parametrize("scale", ["normal", "big"])
def test_random_snapshots(pkg, oracle, L, scale):
    snap = random_snapshot(100 + L, P=333, N=700, G=40, L=L, value_scale=scale, aff=5 if L % 2 else 0)
    res, rows, fit = _run(pkg, snap)
    _check(oracle, snap, res, rows, fit)


@pytest.mark.gpu
def test_all_wide_shape(pkg, oracle):
    """Every lane wide: memory beyond the narrow and scaled ranges on every node and pod."""
    snap = random_snapshot(7, P=200, N=600, G=30, L=9, value_scale="big")
    snap.nodes.alloc[0] = (1 << 40) + np.arange(snap.nodes.n) * 3
    snap.pods.req[0] = np.where(np.arange(snap.pods.n) % 2, (1 << 40) + 1001, 7)
    eng = pkg.Engine(snap.lanes, 0, reasons=True)
    try:
        eng.upload(snap)
        res = eng.evaluate()
        rows, fit, shape = eng.reason_rows(), eng.fit_rows(), eng.fit_shape()
    finally:
        eng.close()
    assert shape["LW"] >= 2
    _check(oracle, snap, res, rows, fit)


@pytest.mark.gpu
@pytest.mark.parametrize("L,d,case", lane_cases.combos())
def test_lane_cases(pkg, oracle, L, d, case):
    snap = lane_cases.lane_snapshot(L, case, d, seed=11)
    res, rows, fit = _run(pkg, snap, fit_bitmap=False)
    _check(oracle, snap, res, rows, None)
    assert rows[:, 4 + d].any()


@pytest.mark.gpu
def test_hand_built_table(pkg, oracle):
    snap = reason_cases.snapshot()
    res, rows, fit = _run(pkg, snap)
    np.testing.assert_array_equal(rows, reason_cases.expected())
    _check(oracle, snap, res, rows, fit)


@pytest.mark.gpu
@pytest.mark.parametrize("aff", [70, 130])
def test_affinity_tables(pkg, oracle, aff):
    """More affinity classes than 64 selector pairs could carry, and pods spread over them."""
    snap = random_snapshot(200 + aff, P=500, N=1100, G=30, L=7, aff=aff)
    res, rows, fit = _run(pkg, snap)
    _check(oracle, snap, res, rows, fit)


@pytest.mark.gpu
@pytest.mark.parametrize("N", [0, 1, 31, 33, 511, 513, 1025])
@pytest.mark.parametrize("P", [1, 37, 70])
def test_unaligned_sizes(pkg, oracle, N, P):
    snap = random_snapshot(N * 7 + P, P=P, N=max(N, 1), G=9, L=6, aff=3)
    if N == 0:
        snap.nodes = snap.nodes.take(np.zeros(0, np.int64))
        snap.aff_bits = None
        snap.pods.aff_class = None
        snap.groups.rep_aff = None
    res, rows, fit = _run(pkg, snap)
    if N == 0:
        assert rows.shape == (P, 10) and not rows.any()
        return
    _check(oracle, snap, res, rows, fit)


MODES = {
    "none": dict(fit_bitmap=False),
    "bitmap": dict(fit_bitmap=True),
    "score+bitmap": dict(fit_bitmap=True, score=True),
    "topk": dict(fit_bitmap=False, topk=8),
    "topk+bitmap+filter": dict(fit_bitmap=True, topk=8, filter=True),
}


def _everything(pkg, snap, reasons, kw):
    eng = pkg.Engine(snap.lanes, 0, reasons=reasons, **kw)
    try:
        eng.upload(snap)
        res = eng.evaluate()
        out = {f: getattr(res, f) for f in ("prefilter", "feasible_count", "best_node", "best_score", "admit",
                                            "admit_bitmap", "new_denied", "order", "rank", "max_group")}
        if kw.get("fit_bitmap"):
            out["fit"] = eng.fit_rows()
        if kw.get("score"):
            out["score"] = eng.score_rows()
        if kw.get("topk"):
            out["topk"] = eng.topk_rows()
        if kw.get("filter"):
            out["filter"] = eng.filter_rows()
            out["filter_code"] = res.filter_code
        rows = eng.reason_rows() if reasons else None
    finally:
        eng.close()
    return out, rows


@pytest.mark.gpu
def test_flag_beside_every_mode(pkg, oracle):
    snap = random_snapshot(301, P=450, N=900, G=40, L=7, aff=4)
    want = fit_reasons_ref.fit_reasons(snap)
    for name, kw in MODES.items():
        base, _ = _everything(pkg, snap, False, kw)
        with_r, rows = _everything(pkg, snap, True, kw)
        for k, v in base.items():
            if isinstance(v, tuple):
                for a, b in zip(v, with_r[k]):
                    np.testing.assert_array_equal(a, b, err_msg=f"{name}: {k}")
            else:
                np.testing.assert_array_equal(v, with_r[k], err_msg=f"{name}: {k}")
        np.testing.assert_array_equal(rows, want, err_msg=name)


@pytest.mark.gpu
def test_row_updates_and_affinity_replacement(pkg, oracle):
    snap = random_snapshot(401, P=400, N=1200, G=40, L=8, aff=6)
    eng = pkg.Engine(snap.lanes, 0, reasons=True)
    try:
        eng.upload(snap)
        res = eng.evaluate()
        _check(oracle, snap, res, eng.reason_rows(), eng.fit_rows())
        rng = np.random.default_rng(401)
        # nodes made unschedulable, labels changed, and the deciding lane moved: cpu freed on some, filled on others
        nidx = np.sort(rng.choice(snap.nodes.n, 40, replace=False))
        nodes = snap.nodes.copy()
        nodes.flags[nidx[:10]] = S.NODE_UNSCHEDULABLE
        nodes.label_mask[nidx[10:20]] ^= np.uint64(0b101)
        nodes.requested[0, nidx[20:30]] = 0
        nodes.requested[0, nidx[30:]] = nodes.alloc[0, nidx[30:]] + 1
        nodes.req_present[nidx[30:]] ^= np.uint32(1 << 5)
        eng.update_nodes(nidx, nodes.take(nidx))
        snap.nodes = nodes
        res = eng.evaluate()
        _check(oracle, snap, res, eng.reason_rows(), eng.fit_rows())
        # group rows change: the rows stay those of the same nodes and pods
        gidx = np.sort(rng.choice(snap.groups.n, 6, replace=False))
        groups = snap.groups.copy()
        groups.matched[gidx] += 1
        groups.flags[gidx] ^= np.uint8(S.GROUP_DENIED)
        eng.update_groups(gidx, groups.take(gidx))
        snap.groups = groups
        res = eng.evaluate()
        _check(oracle, snap, res, eng.reason_rows(), eng.fit_rows())
        # a replaced affinity table
        bits = snap.aff_bits.copy()
        bits ^= rng.integers(0, 1 << 32, bits.shape, dtype=np.uint64).astype(np.uint32)
        W = bits.shape[1]
        bits[:, W - 1] &= np.uint32((1 << (snap.nodes.n % 32)) - 1) if snap.nodes.n % 32 else np.uint32(0xFFFFFFFF)
        eng.upload_affinity(bits)
        snap.aff_bits = bits
        res = eng.evaluate()
        _check(oracle, snap, res, eng.reason_rows(), eng.fit_rows())
    finally:
        eng.close()


@pytest.mark.gpu
def test_full_size_cfg4(pkg, oracle, snapshot_mod):
    snap = snapshot_mod.config(4)
    eng = pkg.Engine(snap.lanes, 0, fit_bitmap=False, reasons=True)
    try:
        eng.upload(snap)
        res = eng.evaluate()
        rows = eng.reason_rows()
    finally:
        eng.close()
    N = snap.nodes.n
    assert rows.shape == (snap.pods.n, 4 + snap.lanes)
    np.testing.assert_array_equal((rows > 0).any(axis=1), res.feasible_count < N)
    idx = np.sort(np.random.default_rng(4).choice(snap.pods.n, 300, replace=False))
    np.testing.assert_array_equal(rows[idx], fit_reasons_ref.fit_reasons(snap, pods=idx))


@pytest.mark.gpu
def test_more_classes_than_a_grid_row(pkg, oracle):
    """70 000 pods with distinct (selector, toleration) classes: the class stage runs in chunks of grid rows."""
    P, N = 70000, 96
    snap = random_snapshot(501, P=P, N=N, G=20, L=5)
    rng = np.random.default_rng(501)
    snap.nodes.label_mask = rng.integers(0, 1 << 20, N).astype(np.uint64)
    snap.pods.sel_mask = np.arange(P, dtype=np.uint64) & np.uint64((1 << 20) - 1)
    snap.pods.tol_mask = (np.arange(P, dtype=np.uint64) >> np.uint64(20)) | np.uint64(1)
    res, rows, fit = _run(pkg, snap, fit_bitmap=False)
    np.testing.assert_array_equal((rows > 0).any(axis=1), res.feasible_count < N)
    idx = np.concatenate([np.arange(300), rng.choice(P, 700, replace=False), np.arange(P - 300, P)])
    np.testing.assert_array_equal(rows[idx], fit_reasons_ref.fit_reasons(snap, pods=idx))


@pytest.mark.gpu
def test_fetch_errors(pkg):
    snap = random_snapshot(601, P=50, N=80, G=5, L=6)
    eng = pkg.Engine(snap.lanes, 0)
    try:
        eng.upload(snap)
        eng.evaluate()
        with pytest.raises(pkg.capi.BsError) as ei:
            eng.reason_rows()
        assert ei.value.code == pkg.capi.BS_E_STATE
    finally:
        eng.close()
    eng = pkg.Engine(snap.lanes, 0, reasons=True)
    try:
        eng.upload(snap)
        with pytest.raises(pkg.capi.BsError) as ei:
            eng.reason_rows()
        assert ei.value.code == pkg.capi.BS_E_STATE
        eng.set_profiling(True)
        eng.evaluate()
        assert eng.reasons_ms() > 0
        assert eng.reason_rows(10, 40).shape == (40, 10)
        for pod0, n in ((0, 51), (50, 1), (49, 2)):
            with pytest.raises(pkg.capi.BsError) as ei:
                eng.reason_rows(pod0, n)
            assert ei.value.code == pkg.capi.BS_E_INDEX
    finally:
        eng.close()


@pytest.mark.gpu
def test_plugin_fit_error():
    binary = native.cpp_program("plugin_reasons_test")
    first, second = json.loads(subprocess.check_output([binary, "reasons"], text=True))
    taints = "1 node(s) had taints that the pod didn't tolerate"
    assert first["lanes"] == second["lanes"] == 5
    assert first["feasible"] == [0, 0, 7]
    assert first["counts"] == [[1, 1, 0, 1, 6, 0, 0, 0, 3], [1, 1, 7, 1, 1, 0, 0, 0, 0], [1, 1, 0, 1, 0, 0, 0, 0, 0]]
    assert first["errors"] == [
        "0/10 nodes are available: " + taints + ", 1 node(s) were unavailable, 1 node(s) were unschedulable, "
        "3 Insufficient nvidia.com/gpu, 6 Insufficient cpu.",
        "0/10 nodes are available: 1 Insufficient cpu, " + taints + ", 1 node(s) were unavailable, "
        "1 node(s) were unschedulable, 7 node(s) didn't match node selector.",
        ""]
    assert first["unknown"] == [0, ""] and second["unknown"] == [0, ""]
    assert second["feasible"] == [1, 0, 8]
    assert second["counts"][0] == [0, 1, 0, 1, 6, 0, 0, 0, 3]
    assert second["errors"] == [
        "",
        "0/10 nodes are available: 1 Insufficient cpu, " + taints + ", 1 node(s) were unavailable, "
        "8 node(s) didn't match node selector.",
        ""]
