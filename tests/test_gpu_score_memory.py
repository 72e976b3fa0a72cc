"""The score matrix's memory (bs_score_memory): compressible device memory where the device supports generic
compression and the driver grants it, cudaMalloc otherwise.  Compression is invisible to readers and writers, so every
round here compares the whole score matrix and fit bitmap with the CPU oracle, bit-exact, in rounds whose elements
span the value classes: rows with no fitting node (all INT64_MIN), narrow scores at the top of their range
(2^27 - 3, the largest a narrow difference reaches), and wide scores with their high words set.  Also: a torch view of
bs_device_buffer(BS_BUF_SCORE) reads what bs_fetch_score_rows returns, growing P moves the matrix to a new allocation,
and closing an engine gives its memory back."""
import ctypes

import numpy as np
import pytest

import fit_shape_cases as fc
from parity import assert_round_equal
from randsnap import random_snapshot

pytestmark = pytest.mark.gpu

I64_MIN = np.iinfo(np.int64).min
CU_DEVICE_ATTRIBUTE_GENERIC_COMPRESSION_SUPPORTED = 107


def _compression_attribute(device=0):
    cu = ctypes.CDLL("libcuda.so.1")
    assert cu.cuInit(0) == 0
    dev, v = ctypes.c_int(), ctypes.c_int()
    assert cu.cuDeviceGet(ctypes.byref(dev), device) == 0
    assert cu.cuDeviceGetAttribute(ctypes.byref(v), CU_DEVICE_ATTRIBUTE_GENERIC_COMPRESSION_SUPPORTED, dev) == 0
    return v.value


def _narrow_top():
    # cfg4's lane shape (3 narrow, 2 scaled); the design drives some pods' narrow minimum to 2^27 - 3
    return fc.shape_snapshot((0, 3, 2), "split")


def _wide_and_empty(seed=9100, P=2999, N=2050):
    # all-wide: residuals up to 2^45, so fitting scores carry high words; every 7th pod asks more than any node has
    snap = random_snapshot(seed, P=P, N=N, G=40, L=5)
    nt, pt = snap.nodes, snap.pods
    rng = np.random.default_rng(seed)
    for d in range(5):
        nt.alloc[d] = rng.integers(1 << 30, 1 << 45, N)
        pt.req[d] = rng.integers(0, 1 << 44, P)
    pt.req[0][::7] = 1 << 46
    return snap


def _evaluate(pkg, snap, eng=None):
    own = eng is None
    eng = eng or pkg.Engine(snap.lanes, 0, fit_bitmap=True, score=True)
    try:
        eng.upload(snap)
        res = eng.evaluate()
        return res, eng.fit_rows(), eng.score_rows(), eng.score_memory(), eng.device_buffer(pkg.capi.BUF_SCORE)
    finally:
        if own:
            eng.close()


def test_reported_memory_matches_device(pkg):
    import torch
    _, _, _, mem, _ = _evaluate(pkg, random_snapshot(9000, P=300, N=200))
    attr = _compression_attribute()
    assert mem["supported"] == attr
    if not attr:
        assert not mem["compressed"]
    if "H100" in torch.cuda.get_device_name(0):
        # the fast path: an H100 supports generic compression and the driver grants it for the score matrix
        assert attr == 1 and mem["compressed"]


@pytest.mark.parametrize("case", ["narrow_top", "wide_and_empty"])
def test_whole_matrices_match_oracle(pkg, oracle, case):
    snap = _narrow_top() if case == "narrow_top" else _wide_and_empty()
    orc = oracle.round(snap, want_bitmap=True, want_score=True)
    assert not orc.ref_panic
    fits = orc.score != I64_MIN
    if case == "narrow_top":
        assert orc.score[fits].max() == (1 << 27) - 3
    else:
        assert (~fits).all(axis=1).any(), "rows with no fitting node"
        assert (orc.score[fits] >> 32 != 0).any(), "wide scores with high words"
    res, fit, sc, mem, _ = _evaluate(pkg, snap)
    assert_round_equal(res, fit, sc, orc)


def test_torch_view_reads_fetched_rows(pkg):
    import torch
    snap = _wide_and_empty(9200, P=1000, N=3001)
    eng = pkg.Engine(snap.lanes, 0, fit_bitmap=False, score=True)
    try:
        eng.upload(snap)
        eng.evaluate()
        ptr, nbytes = eng.device_buffer(pkg.capi.BUF_SCORE)
        pitch = eng.score_pitch()
        assert pitch == 3002 and nbytes == snap.pods.n * pitch * 8

        class _View:
            __cuda_array_interface__ = {"shape": (snap.pods.n, pitch), "typestr": "<i8", "data": (ptr, False),
                                        "version": 3, "strides": None}

        view = torch.as_tensor(_View(), device="cuda")
        torch.cuda.synchronize()
        np.testing.assert_array_equal(view[:, :snap.nodes.n].cpu().numpy(), eng.score_rows())
    finally:
        eng.close()


def test_growing_p_reallocates(pkg, oracle):
    small = random_snapshot(9300, P=500, N=1500)
    big = random_snapshot(9301, P=6000, N=1500)
    eng = pkg.Engine(small.lanes, 0, fit_bitmap=True, score=True)
    try:
        _, _, _, mem0, (_, n0) = _evaluate(pkg, small, eng)
        res, fit, sc, mem1, (_, n1) = _evaluate(pkg, big, eng)
    finally:
        eng.close()
    assert n1 > n0
    assert mem1 == mem0
    assert_round_equal(res, fit, sc, oracle.round(big, want_bitmap=True, want_score=True))


def test_close_returns_memory(pkg):
    import torch
    snap = random_snapshot(9400, P=20000, N=5000)   # an 800 MB score matrix
    _evaluate(pkg, snap)   # loads the engine's kernels: module memory stays for the process
    torch.cuda.synchronize()
    free0, _ = torch.cuda.mem_get_info(0)
    for _ in range(3):
        _evaluate(pkg, snap)
    torch.cuda.synchronize()
    free1, _ = torch.cuda.mem_get_info(0)
    assert abs(free1 - free0) <= 2 << 20, (free0, free1)
