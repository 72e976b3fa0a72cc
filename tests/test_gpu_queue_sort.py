"""The queue sort in every regime it runs in, on the key tables of sort_cases.py: the single-CTA kernel at each of its
size borders, the persistent kernel in its wide and its lean build, tables with more 4096-key tiles than the grid has
CTAs, the radix passes the host drops for constant key bytes, the pass masks across uploads and row updates on one
engine, bs_less, and the refusal of the creation time that is the lister-miss key.

Every round's order and rank are compared exactly with the plain numpy reference (sort_cases.reference), and with the
oracle's round where that is cheap.  No test forces a kernel: each picks table sizes, a node count and output flags so
that the engine's own rule chooses the path, and asserts what bs_sort_shape reports."""
import numpy as np
import pytest

import sort_cases as sc
from parity import run_and_compare
from randsnap import S, random_snapshot

pytestmark = pytest.mark.gpu

SINGLE, LEAN, WIDE = 1, 2, 3
TILE = 4096                     # keys per tile of the persistent kernel
SMALL_MAX = 16384               # the largest table the single-CTA kernel sorts
EDGES = [1, 2, 31, 32, 33, 1023, 1024, 1025, 4095, 4096, 4097, 16383, 16384]
ALL = sorted(sc.CASES)
# the engine sorts beside a fit kernel it estimates at pairs x 0.9 ns without a score or top-K output, and takes the
# lean build above 0.6 ms
LEAN_PAIRS = 0.6 / 0.9e-9


def same(got, exp, what, snap):
    bad = np.flatnonzero(got != exp)
    assert not len(bad), (f"{snap.name} P={snap.pods.n} G={snap.groups.n}: {what} differs at {len(bad)} positions, "
                          f"first {bad[:6].tolist()}: got {got[bad[:6]].tolist()}, expected {exp[bad[:6]].tolist()}")


def check(eng, snap, oracle=None, upload=True):
    """One round of `snap` on `eng`; order and rank against the reference (and the oracle); returns the sort shape."""
    if upload:
        eng.upload_groups(snap.groups)
        eng.upload_pods(snap.pods)
    res = eng.evaluate()
    order, rank = sc.reference(snap.pods, snap.groups)
    same(res.order, order, "order", snap)
    same(res.rank, rank, "rank", snap)
    if oracle is not None:
        orc = oracle.round(snap, want_bitmap=False)
        same(orc.order, order, "oracle order", snap)
        same(orc.rank, rank, "oracle rank", snap)
    return eng.sort_shape()


@pytest.fixture
def engine(pkg):
    """An engine over N empty nodes; closed after the test."""
    made = []

    def make(N=1, **kw):
        eng = pkg.Engine(sc.L, 0, **kw)
        eng.upload_nodes(S.NodeTable.empty(N, sc.L))
        made.append(eng)
        return eng
    yield make
    for eng in made:
        eng.close()


# ---------------------------------------------------------------------------------------------------------------
# the single-CTA kernel

@pytest.mark.parametrize("case", ALL)
def test_single_cta_kernel_at_every_size_border(engine, oracle, case):
    """n = 1, 2, around a warp, around the 1024 threads, around 4 entries per lane, and the last table the kernel
    takes, for the pods; the group count walks the same list out of step, and both are 16384 once."""
    eng = engine()
    sizes = [(P, EDGES[(5 * i + 3) % len(EDGES)]) for i, P in enumerate(EDGES)] + [(SMALL_MAX, SMALL_MAX)]
    for P, G in sizes:
        shape = check(eng, sc.build(case, P, G), oracle)
        assert shape["kernel"] == SINGLE and shape["grid"] == 1, (P, G, shape)


def test_sort_shape_needs_a_round(pkg):
    eng = pkg.Engine(sc.L)
    try:
        with pytest.raises(pkg.capi.BsError) as ei:
            eng.sort_shape()
        assert ei.value.code == pkg.capi.BS_E_STATE
        snap = sc.build("no_groups", 0)
        eng.upload(snap)
        eng.evaluate()
        assert eng.sort_shape() == dict(kernel=0, grid=0, group_passes=0, pod_passes=0)
    finally:
        eng.close()


# ---------------------------------------------------------------------------------------------------------------
# the border between the two kernels

@pytest.mark.parametrize("P,G", [(16385, 100), (100, 16385), (16384, 16385), (16385, 0)])
@pytest.mark.parametrize("case", ["heavy_ties", "group_ties"])
def test_first_tables_of_the_persistent_kernel(engine, oracle, case, P, G):
    """One entry more than the single-CTA kernel takes, in the pods, in the groups alone (a handful of pods, whose
    order shows the group ranks), and without any group."""
    shape = check(engine(), sc.build(case, P, G), oracle)
    assert shape["kernel"] == WIDE and shape["grid"] == (max(P, G) + TILE - 1) // TILE, shape


# ---------------------------------------------------------------------------------------------------------------
# the persistent kernel, wide build: a short fit kernel

@pytest.mark.parametrize("case", ALL)
def test_persistent_wide_build(engine, oracle, case):
    """Six tiles, the last holding one key; two tiles of groups."""
    shape = check(engine(N=8), sc.build(case, 5 * TILE + 1, 5000, N=8), oracle)
    assert shape["kernel"] == WIDE and shape["grid"] == 6, shape


@pytest.mark.parametrize("case", ["heavy_ties", "all_equal", "reversed"])
def test_persistent_wide_build_forty_tiles(engine, oracle, case):
    """More than 32 tiles, the last one key short of full."""
    shape = check(engine(N=8), sc.build(case, 40 * TILE - 1, 9000, N=8), oracle)
    assert shape["kernel"] == WIDE and shape["grid"] == 40, shape


@pytest.mark.parametrize("P,G", [(140000, 2500), (40000, 20000), (17000, 9000)])
def test_queue_sort_table_sizes(pkg, oracle, snapshot_mod, P, G):
    """Compare / queue order (core.go:368-411) across the sort kernel's regimes: more than 32 tiles of 4096 pods
    (tile histograms read from global memory instead of the staged copy), several tiles per table with the
    rank phases reusing a staged tile, and tables just above the single-CTA kernel's limit; ties in every key
    field (few priorities, shared creation times, equal timestamps) so that stability decides the order."""
    rng = np.random.default_rng(P)
    snap = random_snapshot(7700 + G, P=P, N=48, G=G, L=5)
    snap.pods.priority = rng.choice([0, 5, -3], snap.pods.n).astype(np.int32)
    snap.pods.ts_ns = (rng.integers(0, 4000, snap.pods.n) * 1000003 + (1 << 40)).astype(np.int64)
    snap.groups.creation_ns = (rng.integers(0, 300, snap.groups.n) * 7919 + (1 << 33)).astype(np.int64)
    run_and_compare(pkg, oracle, snap, score=False)


# ---------------------------------------------------------------------------------------------------------------
# the persistent kernel, lean build: beside a long fit kernel

def test_persistent_lean_build(engine):
    """40 000 pods x 20 000 nodes without a fit bitmap or scores: 8e8 pairs, which the engine's rule puts above its
    0.6 ms threshold.  The numpy reference alone is the expected answer (the oracle's fit over 8e8 pairs per case
    would take minutes).  Ties decide most of each order, so stability is checked under this build too."""
    P, N = 40_000, 20_000
    assert P * N > LEAN_PAIRS
    eng = engine(N=N, fit_bitmap=False)
    for case in ("heavy_ties", "all_equal", "group_ties", "misses", "ts_only_sign_bit", "ts_extremes", "reversed"):
        shape = check(eng, sc.build(case, P, 6000, N=N))
        assert shape["kernel"] == LEAN and shape["grid"] == 10, (case, shape)


# ---------------------------------------------------------------------------------------------------------------
# more tiles than CTAs: a CTA owns a second tile

def many_tiles():
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return (sms + 9) * TILE + 1, sms + 10


@pytest.mark.parametrize("case,G", [("heavy_ties", 3000), ("all_equal", 1), ("reversed", 3000), ("group_ties", 20000),
                                    ("misses", 3000)])
def test_more_tiles_than_ctas(engine, oracle, case, G):
    """The grid is at most one CTA per SM, so with ten more tiles than SMs the first CTAs run their tile loops twice:
    the shared counters and parked digits are reused, the tiles-before sums run over more tiles than CTAs, and the
    histogram rotation is shared out round-robin.  group_ties has five tiles of groups as well."""
    P, ntiles = many_tiles()
    shape = check(engine(N=8), sc.build(case, P, G, N=8), oracle)
    assert shape["kernel"] == WIDE and shape["grid"] < ntiles, (shape, ntiles)


def test_more_tiles_than_ctas_lean_build(engine):
    """The same under the lean build: about 1300 nodes put P x N above the rule's threshold, still a round of under
    a millisecond of fit work."""
    P, ntiles = many_tiles()
    N = int(1.15 * LEAN_PAIRS / P) + 1
    eng = engine(N=N, fit_bitmap=False)
    for case in ("heavy_ties", "all_equal"):
        shape = check(eng, sc.build(case, P, 3000, N=N))
        assert shape["kernel"] == LEAN and shape["grid"] < ntiles, (case, shape, ntiles)


# ---------------------------------------------------------------------------------------------------------------
# the passes the host keeps: one per key byte that varies.  The pods' second key word always keeps the byte of its
# grouped bit (byte 3), and the bytes of the group ranks 0..G.

PASSES = [
    # case, P, G, group passes, pod passes
    ("all_equal", 5000, 0, 0, 1),             # nothing varies
    ("two_keys_alternating", 5000, 0, 0, 2),  # timestamp byte 2
    ("ts_only_sign_bit", 5000, 0, 0, 2),      # timestamp byte 7
    ("ts_only_byte6", 5000, 0, 0, 2),
    ("ts_extremes", 5000, 0, 0, 9),           # all eight timestamp bytes
    ("prio_extremes", 5000, 0, 0, 5),         # all four priority bytes
    ("groups_all_equal", 5000, 300, 0, None),
    ("one_group", 5000, 1, 0, None),
    ("name_extremes", 5000, 300, 4, None),    # all four name bytes, one creation time
    ("creation_extremes", 5000, 300, 9, None),  # all eight creation bytes and the low name byte
    ("rank_bits", 5000, 255, None, 2),        # ranks 0..255 in byte 0
    ("rank_bits", 5000, 256, None, 3),        # ranks 0..256: byte 1 as well
    ("rank_bits", 5000, 257, None, 3),
    ("ts_only_sign_bit", 5 * TILE + 1, 0, 0, 2),   # the same through the persistent kernel
    ("prio_extremes", 5 * TILE + 1, 0, 0, 5),
    ("rank_bits", 5 * TILE + 1, 257, None, 3),
    ("groups_all_equal", 100, SMALL_MAX + 1, 0, None),
]


@pytest.mark.parametrize("case,P,G,gpass,ppass", PASSES)
def test_constant_bytes_are_skipped_and_the_order_holds(engine, oracle, case, P, G, gpass, ppass):
    shape = check(engine(), sc.build(case, P, G), oracle)
    assert shape["kernel"] == (SINGLE if max(P, G) <= SMALL_MAX else WIDE)
    if gpass is not None:
        assert shape["group_passes"] == gpass, shape
    if ppass is not None:
        assert shape["pod_passes"] == ppass, shape


# ---------------------------------------------------------------------------------------------------------------
# the pass masks across uploads and row updates on one engine

def test_masks_follow_uploads_and_row_updates(engine, oracle):
    eng = engine()
    rng = np.random.default_rng(11)
    P, G = 3000, 200
    base_ts, base_c = sc.T0 & ~0xFF & ~(0xFF << 40), sc.C0 & ~0xFF
    # 1. every key varies in its lowest byte only
    snap = sc.snapshot("low_bytes", 1, rng.integers(0, 2, P), rng.integers(0, G, P), base_ts + rng.integers(0, 200, P),
                        base_c + rng.integers(0, 100, G), rng.integers(0, 50, G))
    shape = check(eng, snap, oracle)
    # groups: creation byte 0, name byte 0; pods: timestamp byte 0, rank byte 0, grouped byte, priority byte 0
    assert (shape["kernel"], shape["group_passes"], shape["pod_passes"]) == (SINGLE, 2, 4), shape
    # 2. new pods whose keys vary in high bytes only: timestamp bytes 5 and 7, priority byte 3
    pt = snap.pods.copy()
    pt.ts_ns = base_ts + (rng.integers(0, 200, P) << 40) + np.where(rng.random(P) < 0.5, sc.INT64_MIN, 0)
    pt.priority = (rng.integers(0, 2, P) << 24).astype(np.int32)
    snap = S.Snapshot(snap.nodes, pt, snap.groups, "high_bytes")
    eng.upload_pods(pt)
    shape = check(eng, snap, oracle, upload=False)
    assert (shape["group_passes"], shape["pod_passes"]) == (2, 5), shape
    # 3. a smaller group table: the pods of groups 50..199 now miss, and their key is 0x7fffffff in the rank bits
    gt = snap.groups.take(np.arange(50))
    snap = S.Snapshot(snap.nodes, pt, gt, "fewer_groups")
    assert (pt.gid >= 50).any()
    eng.upload_groups(gt)
    shape = check(eng, snap, oracle, upload=False)
    assert (shape["group_passes"], shape["pod_passes"]) == (2, 7), shape
    # 4. row updates that bring in a creation byte and a name byte no row had
    idx = np.array([3, 17, 41], np.uint32)
    rows = gt.take(idx)
    rows.creation_ns = rows.creation_ns + np.array([1 << 41, 0, 3 << 41], np.int64)
    rows.name_rank = rows.name_rank + np.array([0, 1 << 17, 1 << 17], np.uint32)
    gt = gt.copy()
    gt.creation_ns[idx], gt.name_rank[idx] = rows.creation_ns, rows.name_rank
    snap = S.Snapshot(snap.nodes, pt, gt, "updated_rows")
    eng.update_groups(idx, rows)
    shape = check(eng, snap, oracle, upload=False)
    assert (shape["group_passes"], shape["pod_passes"]) == (4, 7), shape
    # 5. a large table, a small one, the large one again: the scratch arena is carved anew and the histogram
    #    strides change from round to round
    big, small = sc.build("heavy_ties", 6 * TILE + 77, 5000), sc.build("misses", 500, 40)
    for s, kernel in ((big, WIDE), (small, SINGLE), (big, WIDE), (sc.build("group_ties", 900, 5 * TILE + 3), WIDE)):
        assert check(eng, s, oracle)["kernel"] == kernel, s.name


# ---------------------------------------------------------------------------------------------------------------
# bs_less

def test_less_follows_compare_after_a_persistent_sort(engine, oracle):
    """Compare on sampled pairs: any two pods, two lister misses, a miss and a resolvable pod, grouped and group-less
    pods of one priority, and neighbours in the queue."""
    eng = engine()
    snap = sc.build("misses", 5 * TILE + 1, 300)
    assert check(eng, snap)["kernel"] == WIDE
    pt, gt = snap.pods, snap.groups
    order, _ = sc.reference(pt, gt)
    rng = np.random.default_rng(5)
    grouped = pt.gid != S.GID_NONE
    miss = grouped & ((pt.gid < 0) | (pt.gid >= gt.n) | ((pt.flags & S.POD_LISTER_MISS) != 0))
    pick = lambda mask, n: rng.choice(np.flatnonzero(mask), n)
    same_prio = pt.priority == 0
    at = rng.integers(0, pt.n - 1, 150)
    pairs = np.concatenate([
        rng.integers(0, pt.n, (150, 2)),
        np.stack([pick(miss, 50), pick(miss, 50)], 1),
        np.stack([pick(miss & same_prio, 50), pick(grouped & ~miss & same_prio, 50)], 1),
        np.stack([pick(~grouped & same_prio, 50), pick(grouped & same_prio, 50)], 1),
        np.stack([pick(grouped & ~miss & same_prio, 50), pick(grouped & ~miss & same_prio, 50)], 1),
        np.stack([order[at], order[at + 1]], 1)])
    for a, b in pairs.tolist():
        for x, y in ((a, b), (b, a)):
            assert eng.less(x, y) == oracle.compare(pt, gt, x, y), (x, y, int(pt.gid[x]), int(pt.gid[y]))


# ---------------------------------------------------------------------------------------------------------------
# creation_ns == INT64_MAX is the key of a lister miss: a group may not carry it

def test_creation_int64_max_is_refused(pkg, engine, oracle):
    eng = engine()
    snap = sc.build("creation_extremes", 2000, 60)
    check(eng, snap, oracle)
    bad = snap.groups.copy()
    bad.creation_ns[7] = sc.INT64_MAX
    with pytest.raises(pkg.capi.BsError) as ei:
        eng.upload_groups(bad)
    assert ei.value.code == pkg.capi.BS_E_RANGE
    check(eng, snap, oracle)                      # a valid table again: the round is right
    rows = snap.groups.take([7])
    rows.creation_ns[0] = sc.INT64_MAX
    with pytest.raises(pkg.capi.BsError) as ei:
        eng.update_groups([7], rows)
    assert ei.value.code == pkg.capi.BS_E_RANGE
    check(eng, snap, oracle, upload=False)        # the refused row changed nothing
    rows.creation_ns[0] = sc.INT64_MAX - 1
    eng.update_groups([7], rows)
    snap.groups.creation_ns[7] = sc.INT64_MAX - 1
    check(eng, snap, oracle, upload=False)
