"""The queue-sort key tables on the CPU: the plain numpy reference of Compare's order against the C oracle's round and
the Python restatement, and against Compare itself on sampled pairs; and that each case is the table it claims."""
import time

import numpy as np
import pytest

import pyref
import sort_cases as sc
from randsnap import S

SIZES = [(1, 1), (2, 1), (33, 5), (257, 40), (1500, 257), (4097, 900)]


def check_reference(oracle, snap, restatement=True):
    order, rank = sc.reference(snap.pods, snap.groups)
    P = snap.pods.n
    assert sorted(order.tolist()) == list(range(P))
    orc = oracle.round(snap, want_bitmap=False)
    assert not orc.ref_panic
    np.testing.assert_array_equal(order, orc.order, err_msg="oracle order")
    np.testing.assert_array_equal(rank, orc.rank, err_msg="oracle rank")
    if restatement:
        po, pr = pyref.queue_order(snap.pods, snap.groups)
        np.testing.assert_array_equal(order, po, err_msg="pyref order")
        np.testing.assert_array_equal(rank, pr, err_msg="pyref rank")
    return order, rank


def resolvable(snap):
    """Pods Compare can order: group-less, or in a group the lister finds."""
    gid, G = snap.pods.gid, snap.groups.n
    return (gid == S.GID_NONE) | ((gid >= 0) & (gid < G) & ((snap.pods.flags & S.POD_LISTER_MISS) == 0))


@pytest.mark.parametrize("P,G", SIZES)
@pytest.mark.parametrize("case", sorted(sc.CASES))
def test_reference_agrees_with_oracle_and_pyref(oracle, case, P, G):
    snap = sc.build(case, P, G)
    order, rank = check_reference(oracle, snap)
    # Compare is the rank order wherever both lister lookups succeed
    ok = np.flatnonzero(resolvable(snap))
    if len(ok) >= 2:
        rng = np.random.default_rng(P)
        pairs = rng.choice(ok, (60, 2))
        neighbours = order[np.clip(rng.integers(0, P - 1, 60)[:, None] + [0, 1], 0, P - 1)]
        for a, b in np.concatenate([pairs, neighbours]):
            if resolvable(snap)[a] and resolvable(snap)[b]:
                assert oracle.compare(snap.pods, snap.groups, int(a), int(b)) == bool(rank[a] < rank[b]), (a, b)


@pytest.mark.parametrize("G", [255, 256, 257])
def test_rank_bits_tables(oracle, G):
    snap = sc.build("rank_bits", 2000, G)
    order, rank = check_reference(oracle, snap, restatement=False)
    assert len(np.unique(snap.groups.creation_ns)) == G and set(snap.pods.gid.tolist()) == set(range(G))
    assert rank.max() == G - 1        # one rank per group: the pod ranks are the group ranks


def test_cases_are_the_designed_tables():
    P, G = 3000, 300
    b = lambda case, g=G: sc.build(case, P, g)

    def varying(col):
        u = col.astype(np.int64).view(np.uint64)
        return int(np.bitwise_or.reduce(u) & ~np.bitwise_and.reduce(u))

    o, r = sc.reference(b("all_equal").pods, b("all_equal").groups)
    assert np.array_equal(o, np.arange(P)) and not r.any()
    o, _ = sc.reference(b("two_keys_alternating").pods, b("two_keys_alternating").groups)
    assert np.array_equal(o, np.concatenate([np.arange(1, P, 2), np.arange(0, P, 2)]))
    s = b("sorted")
    assert np.array_equal(sc.reference(s.pods, s.groups)[0], np.arange(P))
    s = b("reversed")
    o, r = sc.reference(s.pods, s.groups)
    assert r[0] == r.max() and r[P - 1] == 0 and (np.diff(r.astype(np.int64)) <= 0).all() and r.max() < P - 1
    assert varying(b("ts_only_sign_bit").pods.ts_ns) == 1 << 63
    assert varying(b("ts_only_byte6").pods.ts_ns) == 0xFF << 48
    assert set(b("ts_extremes").pods.ts_ns.tolist()) == {sc.INT64_MIN, -1, 0, sc.INT64_MAX}
    assert set(b("prio_extremes").pods.priority.tolist()) == {sc.INT32_MIN, -1, 0, sc.INT32_MAX}
    for case in ("ts_only_sign_bit", "ts_only_byte6", "ts_extremes", "prio_extremes", "no_grouped_pods"):
        assert (b(case).pods.gid == S.GID_NONE).all()
    g = b("groups_all_equal").groups
    assert varying(g.creation_ns) == 0 and varying(g.name_rank) == 0
    assert b("one_group").groups.n == 1 and b("no_groups").groups.n == 0
    g = b("group_ties").groups
    assert len(set(zip(g.creation_ns.tolist(), g.name_rank.tolist()))) < G // 2
    assert set(b("creation_extremes").groups.creation_ns.tolist()) == {sc.INT64_MIN, -1, 0, sc.INT64_MAX - 1}
    assert set(b("name_extremes").groups.name_rank.tolist()) == {0, 1, 0xFFFFFFFE, 0xFFFFFFFF}
    m = b("misses")
    assert {S.GID_NONE, S.GID_MISSING, -7, G, G + 5, 0} <= set(m.pods.gid.tolist())
    assert (m.pods.flags & S.POD_LISTER_MISS).any() and m.groups.creation_ns[0] == sc.INT64_MAX - 1
    # group 0's pods sit right in front of the misses of their priority
    o, r = sc.reference(m.pods, m.groups)
    miss = ~resolvable(m)
    for prio in (0, 1):
        in_prio = m.pods.priority == prio
        assert r[in_prio & (m.pods.gid == 0) & ~miss].max() < r[in_prio & miss].min()
        assert r[in_prio & ~miss].max() < r[in_prio & miss].min()


def test_reference_is_fast_enough_for_the_large_cases():
    snap = sc.build("heavy_ties", 700_000, 20_000)
    t = time.perf_counter()
    order, rank = sc.reference(snap.pods, snap.groups)
    dt = time.perf_counter() - t
    assert dt < 2.0, dt
    assert rank[order[0]] == 0 and rank[order[-1]] == rank.max()
