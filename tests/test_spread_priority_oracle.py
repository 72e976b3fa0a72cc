"""CPU: the two restatements of the SelectorSpread priority (tests/spread_priority_ref.c and
tests/pyref_spread_priority.py) agree on random snapshots, alone and with the resource weights, the ratio term and the
node priorities; on the binary64 pins of the blend; on no zones, one zone, and zoned nodes that lie only outside a
pod's fit set; on a non-fitting node that holds the largest count; on Mn = 0 with zones; on pods without a class and
pods that fit no node.  With weight 0 the lists are the existing ones."""
import numpy as np
import pytest

import node_priority_ref as npr
import priority_ref as pr
import pyref_spread_priority as pys
import ratio_priority_ref as rr
import spread_priority_ref as sr
from oracle import oracle
from randsnap import S, random_snapshot

NONE = S.SPREAD_NONE
ZNONE = S.ZONE_NONE


def _agree(snap, nz, K, spread, w, ratio=npr.NO_RATIO, weights=(1, 0, 1), prefs=None, pw=(0, 0)):
    nodes, scores = sr.priority_rows(snap, nz[0], nz[1], K, spread, w, ratio, weights, prefs, pw)
    want = pys.priority_rows(snap, nz[0], nz[1], K, spread, w, ratio, weights, prefs, pw)
    for p, row in enumerate(want):
        assert nodes[p].tolist() == [n for n, _ in row], p
        assert scores[p].tolist() == [s for _, s in row], p
    return nodes, scores


def _fit(snap):
    """[P, N] bool: the fit set of every pod (the oracle's fit bitmap)."""
    bm = oracle.round(snap, want_bitmap=True).fit_bitmap
    bits = np.unpackbits(bm.view(np.uint8), axis=1, bitorder="little")[:, :snap.nodes.n]
    return bits.astype(bool)


def test_binary64_pins():
    # Mn = 50, count = 21, no zones: 100 * (29 / 50) = 57.99999999999999 in binary64
    assert sr.spread_score(50, 21, False, 0, 0) == 57
    assert pys.spread_reduce({0: 21, 1: 50}, {0: None, 1: None})[0] == 57
    # Mn = 4, count = 3, a zoned node whose zone sums 0, Mz = 1..7: 25 / 3 + 200 / 3 = 74.99999999999999 (a node's own
    # count joins its zone's sum, so this one is pinned on the blend itself)
    for mz in range(1, 8):
        assert sr.spread_score(4, 3, True, mz, 0) == 74, mz
        assert pys.node_score(4, 3, True, mz, 0) == 74, mz
    # no selectors: 100 on every node, zoned or not; the blend of 100 and 100 is exactly 100.0
    assert sr.spread_score(0, 0, True, 0, 0) == 100 and sr.spread_score(0, 0, False, 0, 0) == 100
    assert set(pys.spread_reduce({0: 0, 1: 0}, {0: 3, 1: None}).values()) == {100}


@pytest.mark.parametrize("seed", range(5))
@pytest.mark.parametrize("w", [1, 3])
def test_random_snapshots_agree(seed, w):
    snap = random_snapshot(2000 + seed, P=60, N=45, G=8, L=5 + seed % 3)
    nz = S.nonzero_requests(snap, seed)
    spread = S.node_spread(snap, seed, n_zones=[0, 1, 3, 5, 64][seed])
    _agree(snap, nz, 7, spread, w)


@pytest.mark.parametrize("seed", range(3))
@pytest.mark.parametrize("weights", [(1, 0, 1), (2, 3, 5)])
@pytest.mark.parametrize("ratio_on", [False, True])
def test_combined_with_resource_weights_ratio_and_node_priorities(seed, weights, ratio_on):
    snap = random_snapshot(2050 + seed, P=50, N=40, G=6, L=6)
    nz = S.nonzero_requests(snap, seed)
    spread = S.node_spread(snap, seed + 3)
    ratio = (3, rr.BIN_PACK, [1, 1, 0, 0, 2, 1]) if ratio_on else npr.NO_RATIO
    _agree(snap, nz, 9, spread, 1, ratio, weights)
    _agree(snap, nz, 9, spread, 5, ratio, weights, S.node_preferences(snap, seed), (1, 1))


@pytest.mark.parametrize("seed", range(3))
def test_zero_weight_gives_existing_lists(seed):
    snap = random_snapshot(2070 + seed, P=50, N=40, G=6)
    nz = S.nonzero_requests(snap, seed)
    nodes, scores = _agree(snap, nz, 8, S.node_spread(snap, seed), 0)
    n0, s0 = pr.priority_rows(snap, nz[0], nz[1], 8)
    assert np.array_equal(nodes, n0) and np.array_equal(scores, s0)


def test_no_zones_one_zone_and_zones_only_outside_the_fit_set():
    snap = random_snapshot(2080, P=50, N=40, G=6)
    nz = S.nonzero_requests(snap, 4)
    (zone, counts), cls = S.node_spread(snap, 4, occupied=0.6)
    for z in (np.full_like(zone, ZNONE), np.zeros_like(zone)):
        _agree(snap, nz, 10, ((z, counts), cls), 1)
    # zoned nodes only outside a pod's fit set: that pod has no zones, its scores are the node part alone
    fit = _fit(snap)
    n_out = next(n for n in range(snap.nodes.n) if not fit[:, n].all())
    z = np.full_like(zone, ZNONE)
    z[n_out] = 2
    pods = np.nonzero(~fit[:, n_out] & fit.any(axis=1))[0]
    ss = sr.ss_matrix(snap, ((z, counts), cls), pods)
    ss0 = sr.ss_matrix(snap, ((np.full_like(zone, ZNONE), counts), cls), pods)
    assert np.array_equal(ss, ss0)
    _agree(snap, nz, 10, ((z, counts), cls), 1)


def test_non_fitting_node_with_the_largest_count_moves_nothing():
    snap = random_snapshot(2090, P=50, N=40, G=6)
    nz = S.nonzero_requests(snap, 5)
    (zone, counts), cls = S.node_spread(snap, 5, n_zones=3, unzoned=0.0)
    fit = _fit(snap)
    n_out = next(n for n in range(snap.nodes.n) if not fit[:, n].all())
    pods = np.nonzero(~fit[:, n_out] & fit.any(axis=1))[0]
    assert len(pods)
    counts2 = counts.copy()
    counts2[:, n_out] = 1 << 24   # BS_SPREAD_COUNT_MAX
    n0, s0 = _agree(snap, nz, 40, ((zone, counts), cls), 1)
    n2, s2 = _agree(snap, nz, 40, ((zone, counts2), cls), 1)
    assert np.array_equal(n0[pods], n2[pods]) and np.array_equal(s0[pods], s2[pods])


def test_mn_zero_with_zones():
    """Every count 0 on the fit set (Mn = 0, Mz = 0): SS = 100 on every fitting node, zoned or not."""
    snap = random_snapshot(2091, P=40, N=30, G=6)
    nz = S.nonzero_requests(snap, 6)
    (zone, counts), cls = S.node_spread(snap, 6, n_zones=3)
    counts[:] = 0
    ss = sr.ss_matrix(snap, ((zone, counts), cls))
    assert set(np.unique(ss)) <= {-1, 100}
    nodes, scores = _agree(snap, nz, 6, ((zone, counts), cls), 1)
    n0, s0 = pr.priority_rows(snap, nz[0], nz[1], 6)
    assert np.array_equal(nodes, n0) and np.array_equal(scores[nodes >= 0], s0[nodes >= 0] + 100)


def test_pods_without_a_class_score_100():
    snap = random_snapshot(2092, P=40, N=30, G=6)
    nz = S.nonzero_requests(snap, 7)
    (zone, counts), cls = S.node_spread(snap, 7, n_zones=2, occupied=0.8)
    cls[:] = NONE
    nodes, scores = _agree(snap, nz, 6, ((zone, counts), cls), 3)
    n0, s0 = pr.priority_rows(snap, nz[0], nz[1], 6)
    assert np.array_equal(nodes, n0) and np.array_equal(scores[nodes >= 0], s0[nodes >= 0] + 300)


def test_pods_without_fitting_nodes():
    snap = random_snapshot(2093, P=40, N=30, G=6)
    snap.pods.req[0, :10] = 1 << 55   # no node has that much cpu left
    nz = S.nonzero_requests(snap, 8)
    nodes, scores = _agree(snap, nz, 5, S.node_spread(snap, 8), 1)
    assert (nodes[:10] == -1).all() and (scores[:10] == np.iinfo(np.int64).min).all()
