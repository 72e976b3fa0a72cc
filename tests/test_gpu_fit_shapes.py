"""Every instantiated gang_fit lane shape, in every output mode, bit-exact against the CPU oracle, on the designed
rounds of fit_shape_cases.py; and the lane classifier's borders on the device.

Each shape case runs in six configurations (decisions only; the fit bitmap; the score matrix with and without the
bitmap; top-K at K = 5 without the bitmap and at K = 32 with it) at two node counts: N = 1000, one bitmap line, where
every CTA unit sweeps the whole node range; and N = 1100, two lines, where a few pod units (far below 0.9 x the resident
CTA slots of any H100) leave the last wave partial, so the narrow shapes cut their units into node-range pieces and
combine them with the packed (score + 1, ~node) maximum and fit_unpack_kernel.  The engine's lane map (bs_fit_lanes)
must equal the restated classifier's, and the fit stage's launch count must show the path: gang_fit_kernel, plus
fit_unpack_kernel exactly for narrow non-top-K rounds at N = 1100, plus gang_admit_kernel."""
import functools

import numpy as np
import pytest

import fit_shape_cases as fc
from parity import assert_round_equal
from test_gpu_topk import _check_lists

pytestmark = pytest.mark.gpu

SHAPES = fc.instantiated_shapes()
SHAPE_IDS = ["LW{}-LN{}-LS{}".format(*s) for s in SHAPES]
CONFIGS = {
    "none": dict(fit_bitmap=False),
    "bitmap": dict(fit_bitmap=True),
    "score": dict(fit_bitmap=False, score=True),
    "score_bitmap": dict(fit_bitmap=True, score=True),
    "topk5": dict(fit_bitmap=False, topk=5),
    "topk32_bitmap": dict(fit_bitmap=True, topk=32),
}


@functools.lru_cache(maxsize=None)
def _oracle_round(oracle, shape, size):
    snap = fc.shape_snapshot(shape, size)
    orc = oracle.round(snap, want_bitmap=True, want_score=True)
    assert not orc.ref_panic
    return snap, orc


def run(pkg, snap, kw):
    """One profiled round: outputs, lane map, fit_shape and the fit stage's launch count."""
    eng = pkg.Engine(snap.lanes, 0, **kw)
    try:
        eng.set_profiling(True)
        eng.upload(snap)
        out = dict(res=eng.evaluate())
        out["fit"] = eng.fit_rows() if kw.get("fit_bitmap") else None
        out["score"] = eng.score_rows() if kw.get("score") else None
        out["topk"] = eng.topk_rows() if kw.get("topk") else None
        out["lanes"] = eng.fit_lanes()
        out["shape"] = eng.fit_shape()
        out["fit_launches"] = eng.kernel_ms()["gang_fit"][1]
    finally:
        eng.close()
    return out


def check(out, snap, orc, kw):
    kind, unit = fc.classify(snap.nodes, snap.pods)
    assert fc.lane_tokens(*out["lanes"]) == fc.lane_tokens(kind, unit)
    lw, ln, ls = fc.shape_of(kind)
    assert out["shape"] == {"LW": lw, "LN": ln, "LS": ls}
    assert_round_equal(out["res"], out["fit"], out["score"], orc)
    if kw.get("topk"):
        nodes, scores = out["topk"]
        _check_lists(out["res"], nodes, scores, orc.score, kw["topk"])
    return ln


@pytest.mark.parametrize("config", list(CONFIGS))
@pytest.mark.parametrize("size", list(fc.SIZES))
@pytest.mark.parametrize("shape", SHAPES, ids=SHAPE_IDS)
def test_shape(pkg, oracle, shape, size, config):
    snap, orc = _oracle_round(oracle, shape, size)
    kw = CONFIGS[config]
    out = run(pkg, snap, kw)
    ln = check(out, snap, orc, kw)
    assert ln == shape[1]
    split = ln > 0 and not kw.get("topk") and snap.nodes.n > 1024
    assert out["fit_launches"] == 1 + split + (snap.pods.n > 0 and snap.groups.n > 0), out["fit_launches"]


def test_fit_lanes_needs_an_evaluation(pkg):
    snap = fc.shape_snapshot((1, 3, 1), "full")
    eng = pkg.Engine(snap.lanes, 0)
    try:
        eng.upload(snap)
        with pytest.raises(pkg.capi.BsError) as ei:
            eng.fit_lanes()
        assert ei.value.code == pkg.capi.BS_E_STATE
        with pytest.raises(pkg.capi.BsError):
            eng.fit_shape()
    finally:
        eng.close()


@pytest.mark.parametrize("side", [0, 1], ids=["inside", "outside"])
@pytest.mark.parametrize("name", fc.BORDERS)
def test_border(pkg, oracle, name, side):
    snap = fc.border_pair(name)[side]
    kw = CONFIGS["score_bitmap"]
    out = run(pkg, snap, kw)
    assert fc.lane_tokens(*out["lanes"]) == fc.EXPECTED_BORDERS[name][side]
    check(out, snap, oracle.round(snap, want_bitmap=True, want_score=True), kw)


def _evaluate(eng, oracle, nodes, pods, groups, history=()):
    """One round on the engine's current tables: exact against the oracle, and the lane map the statistics give.
    Returns (lane tokens, whether the node tables were prepared again)."""
    snap = fc.S.Snapshot(nodes, pods, groups, "crossing")
    res = eng.evaluate()
    orc = oracle.round(snap, want_bitmap=True, want_score=True)
    assert_round_equal(res, eng.fit_rows(), eng.score_rows(), orc)
    kind, unit = fc.classify(nodes, pods, history)
    got = fc.lane_tokens(*eng.fit_lanes())
    assert got == fc.lane_tokens(kind, unit)
    return got, eng.kernel_ms()["node_left"][0] > 0


def test_engine_crosses_borders(pkg, oracle):
    """One engine across the limits in turn: a pod upload alone changes the lane map (and the node tables are
    prepared again), a row update widens a lane, a row update back leaves it wide (the statistics merge), and a fresh
    node upload narrows it again."""
    base = fc._base()
    nodes, groups = base.nodes, base.groups
    eng = pkg.Engine(base.lanes, 0, fit_bitmap=True, score=True)
    try:
        eng.set_profiling(True)
        eng.upload(base)
        first, prepared = _evaluate(eng, oracle, nodes, base.pods, groups)
        assert prepared and first == "n w s13 n n"
        again, prepared = _evaluate(eng, oracle, nodes, base.pods, groups)
        assert again == first and not prepared
        # a pod beyond the narrow request limit on lane 4
        pods = base.pods.copy()
        pods.req[4, 3] = fc.POD_LIMIT + 1
        eng.upload_pods(pods)
        lanes, prepared = _evaluate(eng, oracle, nodes, pods, groups)
        assert prepared and lanes == "n w s13 n s0"
        # node 7's cpu alloc beyond the narrow node limit: lane 0 leaves the narrow class
        idx = np.array([7], np.uint32)
        edited = nodes.copy()
        edited.alloc[0, 7] = fc.NODE_LIMIT + 1
        eng.update_nodes(idx, edited.take(idx))
        widened, prepared = _evaluate(eng, oracle, edited, pods, groups, history=[nodes])
        assert prepared and widened.split()[0] != "n"
        # the row back as it was: the merged statistics keep the lane wide
        eng.update_nodes(idx, nodes.take(idx))
        kept, _ = _evaluate(eng, oracle, nodes, pods, groups, history=[nodes, edited])
        assert kept == widened
        # a fresh upload narrows it again
        eng.upload_nodes(nodes)
        fresh, prepared = _evaluate(eng, oracle, nodes, pods, groups)
        assert prepared and fresh == lanes
    finally:
        eng.close()
