"""Edges of the fit kernel's score-matrix store path against the CPU oracle, whole matrices compared bit-exact:
odd N (padded score pitch) and a partial last store segment, P not a multiple of the CTA's pod count, tail units
split into node-range pieces that start mid-row, the all-wide and the mixed (wide + narrow + scaled) lane layouts,
and the score matrix with and without the fit bitmap."""
import numpy as np
import pytest

from parity import assert_round_equal
from randsnap import random_snapshot

pytestmark = pytest.mark.gpu


def _mixed(seed, P, N):
    # lane 0 (cpu) narrow, lane 1 (odd memory values above 2^27) wide, lane 2 (multiples of 2^20) scaled
    snap = random_snapshot(seed, P=P, N=N, G=40, L=6)
    nt, pt = snap.nodes, snap.pods
    rng = np.random.default_rng(seed)
    nt.alloc[0] = rng.integers(1000, 64000, N)
    nt.requested[0] = rng.integers(0, 32000, N)
    pt.req[0] = rng.choice([0, 100, 500, 2000, 8000], P)
    nt.alloc[2] = rng.integers(1, 1 << 12, N) << 20
    nt.requested[2] = rng.integers(0, 1 << 11, N) << 20
    pt.req[2] = rng.integers(0, 1 << 10, P) << 20
    return snap


def _all_wide(seed, P, N):
    snap = random_snapshot(seed, P=P, N=N, G=40, L=5)
    nt, pt = snap.nodes, snap.pods
    rng = np.random.default_rng(seed)
    for d in range(5):
        nt.alloc[d] = rng.integers(1 << 30, 1 << 45, N)
        pt.req[d] = rng.integers(0, 1 << 44, P)
    return snap


def _run(pkg, oracle, snap, bitmap):
    eng = pkg.Engine(snap.lanes, 0, fit_bitmap=bitmap, score=True)
    try:
        eng.upload(snap)
        res = eng.evaluate()
        fit = eng.fit_rows() if bitmap else None
        sc = eng.score_rows()
    finally:
        eng.close()
    orc = oracle.round(snap, want_bitmap=True, want_score=True)
    assert not orc.ref_panic
    assert sc.shape == orc.score.shape
    assert_round_equal(res, fit, sc, orc)


# (P, N): 3001 pods = 93 full CTAs of 32 + 25; N = 3001 is odd (pitch 3002) and ends 57 nodes into a store segment;
# a few hundred CTA units leave the last wave partial, so the narrow shapes split it into pieces of whole bitmap
# lines (1024 nodes) that start mid-row; N = 2050 leaves a 2-node last segment in the third line
SHAPES = [(3001, 3001), (2999, 2050), (1000, 4097)]


@pytest.mark.parametrize("P,N", SHAPES)
@pytest.mark.parametrize("bitmap", [True, False])
def test_mixed_lanes_score_matrix(pkg, oracle, P, N, bitmap):
    _run(pkg, oracle, _mixed(7000 + P + N, P, N), bitmap)


@pytest.mark.parametrize("P,N", SHAPES)
@pytest.mark.parametrize("bitmap", [True, False])
def test_all_wide_score_matrix(pkg, oracle, P, N, bitmap):
    _run(pkg, oracle, _all_wide(8000 + P + N, P, N), bitmap)
