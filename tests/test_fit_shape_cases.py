"""CPU: the designed lane-shape rounds of fit_shape_cases.py.  Every shape the gang_fit variant table instantiates has a
case, the restated classifier puts each case on its shape and each border pair on both sides of its limit, and, by
the oracle, each case holds the pairs it was designed for: for every lane class, pairs whose score and whose fit
verdict that class alone decides, differences of -1, 0 and +1 unit, the clamp, the wide high and low words, a narrow
minimum next to 2^27, ties across tiles and absent keys."""
import os
import re

import numpy as np
import pytest

import fit_shape_cases as fc

SHAPES = fc.instantiated_shapes()
SHAPE_IDS = ["LW{}-LN{}-LS{}".format(*s) for s in SHAPES]
ROOT = fc.ROOT


def test_constants_and_variant_table_agree_with_the_sources():
    assert re.search(r"NARROW_LIMIT = \(\(int64_t\)1 << \(FIT_CAP_LOG2 - 1\)\) - 1;", fc.COMMON)
    assert fc.POD_LIMIT == (1 << 26) - 1 and fc.NODE_LIMIT == (1 << 25) - 1 and fc.SCALED_LIMIT == 1 << 29
    inst = open(os.path.join(ROOT, "batch-scheduler_b200", "csrc", "fit_inst.cu")).read()
    wide = {int(a) for a, b in re.findall(r"case (\d+): return pick<(\d+), 0, 0>", inst) if a == b}
    assert wide == set(range(4, fc.MAX_LANES + 1))
    cases = re.findall(r"BS_CASE\((\d+), (\d+)\)", inst.split("#define BS_CASE")[1])
    assert {(int(a), int(b)) for a, b in cases} == set(fc.FIT_WS_COMBOS)
    assert len(SHAPES) == len(set(SHAPES)) == 13 + 78


def test_every_instantiated_shape_has_a_case():
    assert set(fc.SHAPE_CASES) == set(SHAPES)


@pytest.mark.parametrize("shape", SHAPES, ids=SHAPE_IDS)
def test_shape_case_classifies_to_its_shape(shape):
    for size in fc.SIZES:
        snap = fc.shape_snapshot(shape, size)
        kind, unit = fc.classify(snap.nodes, snap.pods)
        assert fc.shape_of(kind) == shape, (size, fc.lane_tokens(kind, unit))
        if shape[1]:
            assert (kind[:4] == fc.NARROW).any()
        assert 0 < snap.pods.n <= 100 and snap.nodes.n == fc.SIZES[size]


def test_lane_classes_move_round_the_lanes():
    seen, units = set(), set()
    for shape in SHAPES:
        snap = fc.shape_snapshot(shape, "full")
        kind, unit = fc.classify(snap.nodes, snap.pods)
        seen |= {(d < 4, int(k)) for d, k in enumerate(kind)}
        units |= {int(u) for k, u in zip(kind, unit) if k == fc.SCALED}
    assert seen == {(f, k) for f in (True, False) for k in (fc.WIDE, fc.NARROW, fc.SCALED)}
    assert {0, 13, fc.FIT_CAP_LOG2, fc.FIT_CAP_LOG2 + 1} <= units


def test_every_border_case_is_a_pair():
    assert set(fc.BORDERS) >= {"alloc_pos", "alloc_neg", "requested_pos", "requested_neg", "pod_count_pos",
                               "pod_count_neg", "pod_req_pos", "pod_req_neg", "pods_lane_pod_count", "scaled_limit_node",
                               "scaled_limit_pos", "scaled_limit_neg", "odd_node", "odd_pod", "odd_node_without_key",
                               "pod_without_key_huge", "float32_rounding", "narrow_cap", "sixteen_narrow",
                               "missing_combo", "missing_combo_walk", "no_fixed_narrow"}


@pytest.mark.parametrize("name", fc.BORDERS)
def test_border_pair_lands_on_both_sides(name):
    inside, outside = fc.border_pair(name)
    want_in, want_out = fc.EXPECTED_BORDERS[name]
    assert want_in != want_out
    assert fc.lane_tokens(*fc.classify(inside.nodes, inside.pods)) == want_in
    assert fc.lane_tokens(*fc.classify(outside.nodes, outside.pods)) == want_out
    for s in (inside, outside):
        assert np.abs(s.nodes.alloc).max() <= fc.VALUE_LIMIT and np.abs(s.nodes.requested).max() <= fc.VALUE_LIMIT
        assert np.abs(s.pods.req).max() <= fc.VALUE_LIMIT


def _decisive(oracle, snap):
    """Per lane class of the case's lane map: what the oracle's round shows about the pairs of that class."""
    kind, unit = fc.classify(snap.nodes, snap.pods)
    orc = oracle.round(snap, want_bitmap=False, want_score=True)
    assert not orc.ref_panic
    score = orc.score
    fit = score != fc.I64_MIN
    diff, class_ok = fc.lane_differences(oracle, snap)
    assert (fit <= class_ok).all()
    # the oracle's fit and score follow from the lane differences
    full = diff.min(axis=0)
    np.testing.assert_array_equal(fit, class_ok & (full >= 0))
    np.testing.assert_array_equal(score[fit], full[fit])
    out = {}
    for c in sorted(set(kind.tolist())):
        lanes = np.flatnonzero(kind == c)
        mc = diff[lanes].min(axis=0)
        mo = diff[np.flatnonzero(kind != c)].min(axis=0) if (kind != c).any() else np.full_like(mc, fc.I64_MAX)
        out[c] = dict(score=(fit & (mc == score) & (mc < mo)).any(),
                      verdict=(~fit & class_ok & (mc < 0) & (mo >= 0)).any(), lanes=lanes)
    return kind, unit, diff, fit, class_ok, score, orc, out


@pytest.mark.parametrize("shape", SHAPES, ids=SHAPE_IDS)
@pytest.mark.parametrize("size", list(fc.SIZES))
def test_shape_case_holds_its_decisive_pairs(oracle, shape, size):
    snap = fc.shape_snapshot(shape, size)
    kind, unit, diff, fit, class_ok, score, orc, out = _decisive(oracle, snap)
    nt, pt = snap.nodes, snap.pods
    for c, o in out.items():
        assert o["score"] and o["verdict"], (c, o)
    for d, tok in enumerate(fc.parse_layout(fc.SHAPE_CASES[shape])):
        u = fc.lane_design(tok, 1)[3]
        others = np.delete(diff, d, axis=0).min(axis=0)
        # -1 unit: only this lane refuses the pair; 0 and +1 unit: fitting pairs
        assert (~fit & class_ok & (diff[d] == -u) & (others >= 0)).any(), (d, tok, "-1")
        assert (fit & (diff[d] == 0)).any() and (fit & (diff[d] == u)).any(), (d, tok)
        if kind[d] == fc.SCALED:
            C = fc.clamp_units(int(unit[d]))
            for m in (C - 1, C, C + 1):
                assert (fit & (diff[d] == m * u)).any(), (d, m)
        if tok == "w":
            assert (fit & (diff[d] >= 1 << 31) & (diff[d] < 1 << 32)).any()
            small = fit & (diff[d] > 1 << 32) & (diff[d] < (1 << 32) + (1 << 27))
            assert small.any() and (not shape[1] or (score[small] < 1 << 27).any())   # the low word alone undercuts them
        if d >= 4:
            bit = np.uint32(1 << d)
            node_has = (((nt.alloc_present & nt.req_present) & bit) != 0)[None, :]
            pod_has = ((pt.req_present & bit) != 0)[:, None]
            assert (fit & ~node_has & pod_has & (pt.req[d] == 0)[:, None]).any(), (d, "node lacks the key")
            assert (fit & node_has & ~pod_has).any(), (d, "pod lacks the key")
    if shape[1]:
        # a narrow minimum next to 2^27: the packed best-node key (score << 4 | word) comes close to 2^31
        assert orc.best_score.max() >= (1 << 27) - 3 and orc.best_score.max() < 1 << 27
        # scores in the clamp's range decided by the narrow lanes (the clamp and the shift back must not undercut them)
        assert ((score > 1 << 26) & (score < 1 << 27)).any()
    # equal best scores in different tiles (and bitmap lines: the tail pieces), won by the lowest node index
    best = orc.best_node
    ties = [p for p in range(pt.n) if best[p] >= 0 and
            len({n // 512 for n in np.flatnonzero(score[p] == orc.best_score[p])}) > 1]
    assert len(ties) >= pt.n // 2
    assert all(best[p] == np.flatnonzero(score[p] == orc.best_score[p])[0] for p in ties)
    if size == "split":
        assert any(np.flatnonzero(score[p] == orc.best_score[p]).max() >= 1024 for p in ties)
