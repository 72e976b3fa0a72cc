"""CPU: the two restatements of the TaintToleration and preferred NodeAffinity priorities (tests/node_priority_ref.c
and tests/pyref_node_priority.py) agree on the normalization's branches, on random snapshots alone and combined with
the resource weights and the ratio term, on pods that fit nowhere, and on the rule that only the fit set sets the
maxima; with both weights 0 the lists are the existing ones."""
import numpy as np
import pytest

import node_priority_ref as npr
import priority_ref as pr
import pyref_node_priority as pyn
import ratio_priority_ref as rr
from oracle import oracle
from randsnap import S, random_snapshot

NONE = S.PREF_NONE


def _agree(snap, nz, K, prefs, pw, ratio=npr.NO_RATIO, weights=(1, 0, 1)):
    nodes, scores = npr.priority_rows(snap, nz[0], nz[1], K, prefs, pw, ratio, weights)
    want = pyn.priority_rows(snap, nz[0], nz[1], K, prefs, pw, ratio, weights)
    for p, row in enumerate(want):
        assert nodes[p].tolist() == [n for n, _ in row], p
        assert scores[p].tolist() == [s for _, s in row], p
    return nodes, scores


def _fit(snap):
    """[P, N] bool: the fit set of every pod (the oracle's fit bitmap)."""
    bm = oracle.round(snap, want_bitmap=True).fit_bitmap
    N = snap.nodes.n
    bits = np.unpackbits(bm.view(np.uint8), axis=1, bitorder="little")[:, :N]
    return bits.astype(bool)


def test_normalize_branches():
    for raw, mx, rev, want in ((0, 0, True, 100), (0, 0, False, 0), (1, 3, True, 67), (2, 3, True, 34),
                               (3, 3, True, 0), (1, 3, False, 33), (2, 3, False, 66), (3, 3, False, 100),
                               ((1 << 31) - 1, (1 << 31) - 1, False, 100), (1, (1 << 31) - 1, False, 0)):
        assert npr.normalize(raw, mx, rev) == want, (raw, mx, rev)
        got = pyn.normalize_reduce({0: raw, 1: mx}, rev)[0]
        assert got == want, (raw, mx, rev)


@pytest.mark.parametrize("seed", range(5))
@pytest.mark.parametrize("pw", [(1, 0), (0, 1), (1, 1), (3, 7)])
def test_random_snapshots_agree(seed, pw):
    snap = random_snapshot(900 + seed, P=60, N=45, G=8, L=5 + seed % 3)
    nz = S.nonzero_requests(snap, seed)
    prefs = S.node_preferences(snap, seed)
    _agree(snap, nz, 7, prefs, pw)


@pytest.mark.parametrize("seed", range(3))
@pytest.mark.parametrize("weights", [(1, 0, 1), (0, 1, 0), (2, 3, 5)])
@pytest.mark.parametrize("ratio_on", [False, True])
def test_combined_with_resource_weights_and_ratio(seed, weights, ratio_on):
    snap = random_snapshot(950 + seed, P=50, N=40, G=6, L=6)
    nz = S.nonzero_requests(snap, seed)
    prefs = S.node_preferences(snap, seed + 7)
    ratio = (3, rr.BIN_PACK, [1, 1, 0, 0, 2, 1]) if ratio_on else npr.NO_RATIO
    _agree(snap, nz, 9, prefs, (1, 1), ratio, weights)
    _agree(snap, nz, 9, prefs, (3, 7), ratio, weights)


@pytest.mark.parametrize("seed", range(3))
def test_zero_weights_give_existing_lists(seed):
    snap = random_snapshot(970 + seed, P=50, N=40, G=6)
    nz = S.nonzero_requests(snap, seed)
    prefs = S.node_preferences(snap, seed)
    nodes, scores = _agree(snap, nz, 8, prefs, (0, 0))
    n0, s0 = pr.priority_rows(snap, nz[0], nz[1], 8)
    assert np.array_equal(nodes, n0) and np.array_equal(scores, s0)


def test_everything_tolerated_gives_100_and_no_class_gives_0():
    snap = random_snapshot(980, P=40, N=30, G=6)
    nz = S.nonzero_requests(snap, 1)
    taints, table, _, _ = S.node_preferences(snap, 1, tainted=1.0)
    tol = np.full(snap.pods.n, np.uint64(0xFFFFFFFFFFFFFFFF))
    cls = np.full(snap.pods.n, NONE, np.uint32)
    prefs = (taints, table, tol, cls)
    assert (npr.maxima(snap, prefs) == 0).all()   # Mt = 0 and Ma = 0 for every pod
    nodes, scores = _agree(snap, nz, 6, prefs, (1, 1))
    n0, s0 = pr.priority_rows(snap, nz[0], nz[1], 6)
    assert np.array_equal(nodes, n0)
    assert np.array_equal(scores[nodes >= 0], s0[nodes >= 0] + 100)   # TT = 100 everywhere, NA = 0


def test_pods_without_fitting_nodes():
    snap = random_snapshot(981, P=40, N=30, G=6)
    snap.pods.req[0, :10] = 1 << 55   # no node has that much cpu left
    nz = S.nonzero_requests(snap, 2)
    prefs = S.node_preferences(snap, 2)
    assert (npr.maxima(snap, prefs, pods=range(10)) == 0).all()
    nodes, scores = _agree(snap, nz, 5, prefs, (1, 1))
    assert (nodes[:10] == -1).all() and (scores[:10] == np.iinfo(np.int64).min).all()


@pytest.mark.parametrize("seed", range(3))
def test_non_fitting_node_does_not_move_the_maxima(seed):
    """A node outside a pod's fit set with a raw count above every fitting node's changes no score of that pod."""
    snap = random_snapshot(990 + seed, P=50, N=40, G=6)
    nz = S.nonzero_requests(snap, seed)
    taints, table, tol, cls = S.node_preferences(snap, seed, n_bits=8, tolerate=0.2, tolerate_all=0.0)
    fit = _fit(snap)
    outside = [n for n in range(snap.nodes.n) if not fit[:, n].all()]
    assert outside
    n_out = outside[0]
    pods = np.nonzero(~fit[:, n_out] & fit.any(axis=1))[0]
    assert len(pods)
    # the node outside the fit sets of `pods` gets every taint and a weight above every other node's
    taints2, table2 = taints.copy(), table.copy()
    taints2[n_out] = np.uint64(0xFF)
    table2[:, n_out] = table.max() * 10 + 1000
    tol2 = np.zeros_like(tol)   # nothing tolerated: the node's 8 taints all count
    prefs0 = (taints, table, tol2, cls)
    prefs2 = (taints2, table2, tol2, cls)
    n0, s0 = _agree(snap, nz, 40, prefs0, (1, 1))
    n2, s2 = _agree(snap, nz, 40, prefs2, (1, 1))
    assert np.array_equal(n0[pods], n2[pods]) and np.array_equal(s0[pods], s2[pods])
    assert np.array_equal(npr.maxima(snap, prefs0, pods), npr.maxima(snap, prefs2, pods))
    # it does move the maxima of the pods it fits (the change is visible where it should be)
    fits_out = np.nonzero(fit[:, n_out])[0]
    if len(fits_out):
        assert (npr.maxima(snap, prefs2, fits_out)[:, 0] == 8).all()
