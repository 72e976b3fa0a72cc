"""Key tables for the queue sort, and a plain reference of the order it must produce.

ScheduleOperation.Compare (core.go:368-411) orders the queue by a lexicographic key: priority descending, group-less
pods before grouped ones, PodGroup creation ascending, group name descending, queue timestamp ascending; equal keys
keep table order.  A grouped pod whose lister lookup fails (an unknown group index, or POD_LISTER_MISS) sorts after
every resolvable group of its priority: creation INT64_MAX, name rank 0 (oracle/bs_oracle.c:key_less).  rank is the
number of key changes before a pod along the order.

The engine sorts by radix passes over the key bytes that vary over the table, in one of three kernels chosen by the
table sizes.  Random snapshots vary the same few low bytes every time, so each case here sets the key columns on
purpose: one varying byte in an unusual place, the extremes of every field, ties that only stability can order, and
every way a pod can miss its group.  Requests and nodes play no part: the node table is `N` empty nodes.
"""
from __future__ import annotations

import numpy as np

from randsnap import S

INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
INT32_MIN, INT32_MAX = -(1 << 31), (1 << 31) - 1
T0 = 1_700_000_000 * 10**9          # a queue timestamp
C0 = 1_600_000_000 * 10**9          # a creation time
L = 4


# ---------------------------------------------------------------------------------------------------------------
# the reference

def reference(pt, gt):
    """(order, rank) of the pod table by Compare's key, from the rule above: one stable lexicographic sort of the
    key columns.  Every column is int64 and no negation can wrap (priority and name rank are 32-bit)."""
    P, G = pt.n, gt.n
    gid = pt.gid.astype(np.int64)
    grouped = gid != S.GID_NONE
    miss = grouped & ((gid < 0) | (gid >= G) | ((pt.flags & S.POD_LISTER_MISS) != 0))
    found = grouped & ~miss
    g = np.where(found, gid, 0)
    creation = gt.creation_ns[g] if G else np.zeros(P, np.int64)
    name = gt.name_rank[g].astype(np.int64) if G else np.zeros(P, np.int64)
    creation = np.where(found, creation, np.where(miss, INT64_MAX, 0))
    name = np.where(found, name, 0)
    cols = (-pt.priority.astype(np.int64), grouped.astype(np.int64), creation, -name, pt.ts_ns)
    order = np.lexsort(cols[::-1])                  # stable; the last key given is the most significant
    change = np.zeros(P, bool)
    for c in cols:
        s = c[order]
        change[1:] |= s[1:] != s[:-1]
    rank = np.zeros(P, np.uint32)
    rank[order] = np.cumsum(change)
    return order.astype(np.uint32), rank


# ---------------------------------------------------------------------------------------------------------------
# builders

def snapshot(name, N, prio, gid, ts, creation, name_rank, pflags=None):
    """A snapshot of N empty nodes with the given key columns; scalars are broadcast over the pods."""
    P, G = len(gid), len(creation)
    nt = S.NodeTable.empty(N, L)
    gt = S.GroupTable.empty(G, L)
    gt.min_member[:] = 1
    gt.flags[:] = S.GROUP_HAS_POD | S.GROUP_HAS_MINRES
    gt.creation_ns = np.asarray(creation, np.int64)
    gt.name_rank = np.asarray(name_rank, np.uint32)
    pt = S.PodTable.empty(P, L)
    pt.priority = np.broadcast_to(np.asarray(prio, np.int32), (P,)).copy()
    pt.gid = np.asarray(gid, np.int32)
    pt.ts_ns = np.broadcast_to(np.asarray(ts, np.int64), (P,)).copy()
    if pflags is not None:
        pt.flags = np.asarray(pflags, np.uint8)
    return S.Snapshot(nt, pt, gt, name)


def _filler_groups(G):
    """A group table no case depends on: one creation time, one name."""
    return np.full(G, C0, np.int64), np.full(G, 5, np.uint32)


def _none(P):
    return np.full(P, S.GID_NONE, np.int32)


def _mixed_gid(rng, P, G, none=0.1, missing=0.03):
    gid = rng.integers(0, G, P) if G else np.full(P, S.GID_NONE)
    u = rng.random(P)
    return np.where(u < none, S.GID_NONE, np.where(u < none + missing, S.GID_MISSING, gid)).astype(np.int32)


def all_equal(P, G, N, rng):
    """Every pod has the same key (all in group 0 when there is one): the order is the identity, every rank 0."""
    gid = np.zeros(P, np.int32) if G else _none(P)
    return snapshot("all_equal", N, 7, gid, T0, *_filler_groups(G))


def two_keys_alternating(P, G, N, rng):
    """Even pods carry the later of two timestamps: the odd pods come first, each half in table order."""
    gid = np.zeros(P, np.int32) if G else _none(P)
    ts = T0 + np.where(np.arange(P) % 2 == 0, 1 << 16, 0)
    return snapshot("two_keys_alternating", N, 7, gid, ts, *_filler_groups(G))


def heavy_ties(P, G, N, rng):
    """Three priorities, a few hundred creation times and a few thousand timestamps, duplicate names, a tenth of
    the pods group-less and a few in a missing group: ties in every field, the filler of the size sweeps."""
    prio = rng.choice([0, 5, -3], P)
    ts = rng.integers(0, 4000, P) * 1000003 + (1 << 40)
    creation = rng.integers(0, 300, G) * 7919 + (1 << 33)
    names = rng.integers(0, max(2, G // 2), G)
    return snapshot("heavy_ties", N, prio, _mixed_gid(rng, P, G), ts, creation, names)


def _reordered(snap, name, reverse):
    order, _ = reference(snap.pods, snap.groups)
    return S.Snapshot(snap.nodes, snap.pods.take(order[::-1] if reverse else order), snap.groups, name)


def sorted_(P, G, N, rng):
    """heavy_ties with the pod table already in queue order."""
    return _reordered(heavy_ties(P, G, N, rng), "sorted", False)


def reversed_(P, G, N, rng):
    """heavy_ties with the pod table in reverse queue order: every pod moves, and equal keys swap back."""
    return _reordered(heavy_ties(P, G, N, rng), "reversed", True)


TS_SIGN_BASE = 0x123456789ABCDEF0


def ts_only_sign_bit(P, G, N, rng):
    """Timestamps c and c + INT64_MIN: only bit 63 differs.  One priority, no grouped pod."""
    ts = np.where(rng.random(P) < 0.5, TS_SIGN_BASE, TS_SIGN_BASE + INT64_MIN)
    return snapshot("ts_only_sign_bit", N, 3, _none(P), ts, *_filler_groups(G))


def ts_extremes(P, G, N, rng):
    """Timestamps INT64_MIN, -1, 0 and INT64_MAX."""
    ts = rng.choice(np.array([INT64_MIN, -1, 0, INT64_MAX], np.int64), P)
    return snapshot("ts_extremes", N, 3, _none(P), ts, *_filler_groups(G))


def ts_only_byte6(P, G, N, rng):
    """Timestamps that differ in byte 6 alone."""
    ts = (T0 & ~(0xFF << 48)) + (rng.integers(0, 256, P) << 48)
    return snapshot("ts_only_byte6", N, 3, _none(P), ts, *_filler_groups(G))


def prio_extremes(P, G, N, rng):
    """Priorities INT32_MIN, -1, 0 and INT32_MAX, one timestamp: table order decides inside a priority."""
    prio = rng.choice(np.array([INT32_MIN, -1, 0, INT32_MAX], np.int64), P)
    return snapshot("prio_extremes", N, prio, _none(P), T0, *_filler_groups(G))


def groups_all_equal(P, G, N, rng):
    """One creation time and one name over the group table: every group rank is 0 and the group sort has no pass;
    the grouped pods order by timestamp, then index."""
    ts = T0 + rng.integers(0, 7, P) * 1000
    return snapshot("groups_all_equal", N, 3, _mixed_gid(rng, P, G, none=0.2, missing=0.0), ts, *_filler_groups(G))


def one_group(P, G, N, rng):
    """A table of one group; `G` is ignored."""
    gid = np.where(rng.random(P) < 0.5, 0, S.GID_NONE)
    ts = T0 + rng.integers(0, 50, P) * 1000
    return snapshot("one_group", N, rng.choice([0, 1], P), gid, ts, [C0], [9])


def group_ties(P, G, N, rng):
    """Many groups share (creation, name): their pods interleave by timestamp, then index."""
    k = max(1, G // 8)
    creation = C0 + rng.integers(0, max(1, k // 2), G) * 10**9
    names = rng.integers(0, 3, G)
    ts = T0 + rng.integers(0, 20, P) * 1000
    return snapshot("group_ties", N, rng.choice([0, 1], P), _mixed_gid(rng, P, G, none=0.05, missing=0.0), ts,
                     creation, names)


def creation_extremes(P, G, N, rng):
    """Creation times INT64_MIN, -1, 0 and INT64_MAX - 1 (INT64_MAX itself is refused: it is the miss key)."""
    creation = rng.choice(np.array([INT64_MIN, -1, 0, INT64_MAX - 1], np.int64), G)
    ts = T0 + rng.integers(0, 20, P) * 1000
    return snapshot("creation_extremes", N, 3, _mixed_gid(rng, P, G), ts, creation, rng.integers(0, 3, G))


def name_extremes(P, G, N, rng):
    """Name ranks 0, 1, 0xFFFFFFFE and 0xFFFFFFFF under one creation time."""
    names = rng.choice(np.array([0, 1, 0xFFFFFFFE, 0xFFFFFFFF], np.int64), G)
    ts = T0 + rng.integers(0, 20, P) * 1000
    return snapshot("name_extremes", N, 3, _mixed_gid(rng, P, G), ts, np.full(G, C0, np.int64), names)


def misses(P, G, N, rng):
    """Every way to have no group or to miss it: GID_NONE, GID_MISSING, another negative index, index G, index G + 5
    and POD_LISTER_MISS on a valid index, among resolvable pods.  Group 0 was created at INT64_MAX - 1 with name
    rank 0: its key is one below the misses', so only its group rank keeps its pods in front of them."""
    G = max(G, 1)
    creation = C0 + rng.integers(0, 5, G) * 10**9
    names = rng.integers(0, 3, G)
    creation[0], names[0] = INT64_MAX - 1, 0
    kind = rng.integers(0, 9, P)
    valid = rng.integers(0, G, P)
    gid = np.select([kind == 0, kind == 1, kind == 2, kind == 3, kind == 4, kind == 5],
                    [S.GID_NONE, S.GID_MISSING, -7, G, G + 5, 0], valid)
    pflags = np.where(kind == 6, S.POD_LISTER_MISS, 0)
    ts = T0 + rng.integers(0, 6, P) * 1000
    return snapshot("misses", N, rng.choice([0, 1], P), gid, ts, creation, names, pflags)


def no_grouped_pods(P, G, N, rng):
    """A group table with varied keys that no pod refers to."""
    creation = C0 + rng.integers(0, 1 << 40, G)
    ts = T0 + rng.integers(0, 300, P) * 1000
    return snapshot("no_grouped_pods", N, rng.choice([0, 5, -3], P), _none(P), ts, creation, np.arange(G))


def no_groups(P, G, N, rng):
    """An empty group table (`G` is ignored): every pod is group-less or misses."""
    gid = rng.choice(np.array([S.GID_NONE, S.GID_NONE, S.GID_MISSING, 0, 3]), P)
    ts = T0 + rng.integers(0, 300, P) * 1000
    return snapshot("no_groups", N, rng.choice([0, 5, -3], P), gid, ts, [], [])


def rank_bits(P, G, N, rng):
    """All creation times distinct, one priority, one timestamp: the group ranks are 0..G-1 and alone decide the
    order of the grouped pods.  With G = 255, 256, 257 the top rank sits at a byte border of the bits the pod sort
    keeps for group ranks.  Every group has a pod when P >= G."""
    creation = C0 + rng.permutation(G).astype(np.int64) * 1000
    gid = np.concatenate([np.arange(min(P, G)), rng.integers(0, max(G, 1), max(P - G, 0))]) if G else _none(P)
    rng.shuffle(gid)
    return snapshot("rank_bits", N, 3, gid, T0, creation, np.zeros(G, np.uint32))


CASES = {f.__name__.rstrip("_"): f for f in (
    all_equal, two_keys_alternating, sorted_, reversed_, ts_only_sign_bit, ts_extremes, ts_only_byte6, prio_extremes,
    groups_all_equal, one_group, group_ties, creation_extremes, name_extremes, misses, no_grouped_pods, no_groups,
    rank_bits, heavy_ties)}

# cases whose group table has exactly the size asked for and whose pods refer to it: worth a sweep over G
GROUPED = ("all_equal", "sorted", "reversed", "groups_all_equal", "group_ties", "creation_extremes", "name_extremes",
           "misses", "rank_bits", "heavy_ties")


def build(case, P, G=0, N=1, seed=0):
    """The named case with P pods, G groups (where the case takes a size) and N empty nodes."""
    rng = np.random.default_rng([seed, P, G, sorted(CASES).index(case)])
    return CASES[case](P, G, N, rng)
