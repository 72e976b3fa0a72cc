"""The designed lane-count rounds of lane_cases.py on the CPU: the oracle agrees with the pure-Python restatement on
every lane count and deciding lane, and the deciding lane really decides, so that the GPU parity tests of
test_gpu_lane_counts.py would see a kernel that drops or misreads it."""
import numpy as np
import pytest

import lane_cases as lc
import pyref

LANE_PAIRS = [(L, d) for L in lc.LANES for d in lc.deciding_lanes(L)]


@pytest.mark.parametrize("L,d", LANE_PAIRS)
def test_oracle_matches_python_restatement(oracle, L, d):
    for case in lc.CASES:
        snap = lc.small_snapshot(L, case, d, seed=5)
        r = oracle.round(snap, want_bitmap=True, want_score=True, want_filter=True)
        codes, denied, m = pyref.prefilter_round(snap)
        assert r.max_group == m
        np.testing.assert_array_equal(r.prefilter, codes)
        np.testing.assert_array_equal(r.new_denied, denied)
        py = pyref.round_outputs(snap)
        bits = np.unpackbits(r.fit_bitmap.view(np.uint8), axis=1, bitorder="little")[:, :snap.nodes.n].astype(bool)
        np.testing.assert_array_equal(bits, py["fit"])
        np.testing.assert_array_equal(r.score, py["score"])
        for k in ("feasible_count", "best_node", "best_score", "admit", "order", "rank"):
            np.testing.assert_array_equal(getattr(r, k), py[k], err_msg=k)
        passes, fcodes = pyref.filter_round(snap)
        fbits = np.unpackbits(r.filter_bitmap.view(np.uint8), axis=1, bitorder="little")[:, :snap.nodes.n]
        np.testing.assert_array_equal(r.filter_code, fcodes)
        np.testing.assert_array_equal(fbits.astype(bool), passes)
        nodes = [pyref.Node(snap.nodes, i) for i in range(snap.nodes.n)]
        for sel in (lc.CLS_ALL, lc.CLS_LOW):
            for pct in (1.0, 0.7):
                need, npres = lc.cluster_needs(snap, d, sel, pct, n=12)
                got = lc.cluster_answers(oracle, snap, need, npres, sel, pct)
                exp = [pyref.compare_cluster(nodes, sel, 0, pyref.resource_from(need[:, j], npres[j], L), pct)
                       for j in range(need.shape[1])]
                np.testing.assert_array_equal(got, exp)
        queue = np.random.default_rng(L).permutation(snap.pods.n)
        pf, node, ready, _ = oracle.replay(snap, queue)
        a, b, c = pyref.replay(snap, queue)
        np.testing.assert_array_equal(pf, a)
        np.testing.assert_array_equal(node, b)
        np.testing.assert_array_equal(ready, c)


@pytest.mark.parametrize("L,d,case", lc.combos())
def test_the_deciding_lane_decides(oracle, L, d, case):
    """Without the lane, and with the node side's values moved to the neighbouring lane, the oracle's outputs change
    in many entries.  Exceptions, by design: in case B the max group asks for the deciding lane, so Filter's case 3
    passes every node either way; Filter reads no scalar lane of a node (getLeftResource), so the node-side swap
    cannot reach it; and in "mixed" only the pods of the absent-key class pass PreFilter, whose walk the swap
    seldom changes."""
    snap = lc.lane_snapshot(L, case, d, seed=1)
    base = lc.oracle_outputs(oracle, snap, d)
    off = lc.changed_entries(base, lc.oracle_outputs(oracle, lc.lane_insensitive(snap, d), d, need_lane=False))
    want = dict(prefilter=20, fit=100_000, filter=20_000 if case != "B" else 0, cluster=20, replay=10)
    assert all(off[k] >= v for k, v in want.items()), (off, want)
    nb = lc.neighbour(d, L)
    moved = lc.changed_entries(base, lc.oracle_outputs(oracle, lc.swap_node_lanes(snap, d, nb), d))
    want = dict(prefilter=3, fit=1000 if d >= 4 else 0, cluster=20, replay=1 if case != "mixed" else 0)
    assert all(moved[k] >= v for k, v in want.items()), (nb, moved, want)


def test_every_lane_count_and_build_is_covered():
    Ls = {L for L, _, _ in lc.combos()}
    assert Ls == set(range(4, 17))
    assert all(lc.deciding_lanes(L) == ([3] if L == 4 else [4] if L == 5 else [4, L - 1]) for L in Ls)
    snap = lc.lane_snapshot(7, "A", 6, seed=1)
    assert snap.nodes.n > 2 * 1024 and snap.pods.n % 32 != 0
    kinds = (snap.nodes.alloc_present >> 6) & 1, (snap.nodes.req_present >> 6) & 1
    assert ((kinds[0] & kinds[1]) == 1).any() and ((kinds[0] & kinds[1]) == 0).any()
    assert (snap.nodes.flags != 0).sum() >= 40
