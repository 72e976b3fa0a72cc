"""Designed cases for bs_replay / bs_replay_priority: one per regime the walk's fast paths change (replay.cuh).

Each case is a snapshot, a queue and the regime the walk must land in: the values bs_replay_shape reports, restated
here from replay_walk's host rule (`regime`) and from the kernel's `lo` / `monotone`.  Every case also names the
property it was built for; tests/test_replay_regime_cases.py checks each property on the CPU with the oracle, and
tests/test_gpu_replay_regimes.py runs every case on the device against the oracle and the restatement of
bs_replay_priority.  The snapshots start from randsnap.random_snapshot and are edited into shape."""
from __future__ import annotations

import functools
from dataclasses import dataclass, field

import numpy as np

from randsnap import S, random_snapshot

BLOCK = 1024              # nodes per scan block (REPLAY_BLOCK)
MAX_BLOCKS = 1024         # blocks the summary cache can index
MAX_CLASSES = 32          # representative classes with a checkFit bit
MAX_BUCKETS = 1024        # findMaxPG buckets
UNFIT_SEL = 1 << 8        # a selector bit no node label carries (randsnap labels are 0..15)


@dataclass
class Case:
    name: str
    snap: object
    queue: np.ndarray
    regime: dict                                   # bs_replay_shape values the walk must report
    info: dict = field(default_factory=dict)       # what the CPU test checks the design against
    priority: bool = True                          # also run bs_replay_priority against its restatement
    panic_at: int | None = None                    # first queue position where findMaxPG divides by zero


def rep_classes(snap) -> int:
    """Representative classes of a freshly uploaded engine: distinct (sel, tol, affinity) over pods and groups."""
    pt, gt = snap.pods, snap.groups
    pa = pt.aff_class if pt.aff_class is not None else np.full(pt.n, S.AFF_NONE, np.uint32)
    ga = getattr(gt, "rep_aff", None)
    ga = ga if ga is not None else np.full(gt.n, S.AFF_NONE, np.uint32)
    keys = set(zip(pt.sel_mask.tolist(), pt.tol_mask.tolist(), pa.tolist()))
    keys |= set(zip(gt.rep_sel.tolist(), gt.rep_tol.tolist(), ga.tolist()))
    return max(len(keys), 1)


def safe(snap, n_queue: int) -> bool:
    """replay_walk's bound on the block cache's running sums (every one below 2^62), in exact integers."""
    nt, pt = snap.nodes, snap.pods
    absmax = lambda a: int(np.abs(a).max()) if a.size else 0
    pc = absmax(nt.pod_count.astype(np.int64))
    worst = 0
    for d in range(nt.lanes):
        neg = max(0, -int(pt.req[d].min())) if pt.n else 0
        req = max(int(pt.req[d].max()) if pt.n else 0, 0, neg)
        worst = max(worst, absmax(nt.alloc[d]) + absmax(nt.requested[d]) + req + neg * n_queue + pc + n_queue)
    return worst * max(nt.n, 1) < 4 * 10**18


def buckets(G: int):
    """findMaxPG's bucket size S and count NB (replay.cuh)."""
    per = -(-G // (32 * MAX_BUCKETS))
    size = 32 * max(per, 1)
    return size, -(-G // size)


def regime(snap, n_queue: int) -> dict:
    """What bs_replay_shape reports for a walk of n_queue pods on a freshly uploaded engine, except `lo`."""
    n_rep = rep_classes(snap)
    n_blocks = -(-snap.nodes.n // BLOCK)
    fitmask = n_rep <= MAX_CLASSES
    size, nb = buckets(snap.groups.n)
    pt = snap.pods
    monotone = pt.n == 0 or all(int(pt.req[d].min()) >= 0 for d in (S.LANE_CPU, S.LANE_MEM, S.LANE_EPH))
    return dict(cached=int(safe(snap, n_queue) and fitmask and 1 <= n_blocks <= MAX_BLOCKS), fitmask=int(fitmask),
                n_rep=n_rep, n_blocks=n_blocks, bucket_size=size, n_buckets=nb, monotone=int(monotone))


def _clean_nodes(nt, cpu_alloc, cpu_requested):
    """Every node visible, fitting every selector / toleration, with room on every lane but cpu, as given."""
    N = nt.n
    nt.flags[:] = 0
    nt.label_mask[:] = 0xF
    nt.taint_mask[:] = 0
    nt.alloc[0], nt.requested[0] = cpu_alloc, cpu_requested
    nt.alloc[1], nt.requested[1] = 1 << 34, np.arange(N) % 7 << 20
    nt.alloc[2], nt.requested[2] = 1 << 36, 0
    nt.alloc[3], nt.requested[3] = 110, 0
    nt.pod_count[:] = np.arange(N) % 5


def _walkable_groups(gt):
    gt.flags &= ~np.uint8(S.GROUP_DENIED | S.GROUP_SCHEDULED)


# ---- cache limits ----
CACHE_N = MAX_BLOCKS * BLOCK                     # 1 048 576: the last node the cache can index


def cache_limit(N: int, case: str, seed: int = 7) -> Case:
    """The first N - 1024 nodes leave exactly nothing on the cpu lane at the walk's percent (1.0 for case A, 0.7 for
    case B), the last 1024 have room: a need larger than one node is first met in the last block, where every pod
    is then assumed, so that block's summary goes stale over and over."""
    from oracle import oracle
    pct = 1.0 if case == "A" else 0.7
    snap = random_snapshot(seed, P=40, N=N, G=12, L=5, case=case)
    nt = snap.nodes
    head = N - BLOCK
    zero = oracle.scale(4000, pct)                 # requested = scale(alloc, pct): residual 0 at pct
    _clean_nodes(nt, np.where(np.arange(N) < head, 4000, 64000), np.where(np.arange(N) < head, zero, 1000))
    gt = snap.groups
    _walkable_groups(gt)
    gt.flags |= S.GROUP_HAS_POD | S.GROUP_HAS_MINRES
    gt.min_member[:] = 4
    gt.scheduled[:] = 0
    gt.min_res[0] = 8_000_000                      # 4 x 8M cpu: about half the last block
    gt.min_res[1:3] = 0
    gt.min_res[4] = 0
    gt.min_res_present[:] = 0
    pt = snap.pods
    pt.req[0] = np.maximum(pt.req[0], 2000)         # no pod fits the head, where 1200 cpu is left at most
    pt.req[1] = np.minimum(pt.req[1], 1 << 30)
    pt.req_present[:] = 0                           # the need is on the fixed lanes only
    q = np.arange(pt.n, dtype=np.uint32)
    info = dict(head=head, percent=pct)
    reg = dict(cached=int(N <= CACHE_N), fitmask=1, n_blocks=-(-N // BLOCK))
    return Case(f"cache_{case}_N{N}", snap, q, reg, info)


def big_values(N: int, seed: int = 11) -> Case:
    """value_scale="big": memory near 2^55 takes the running sums past the cache's bound, so the walk scans
    block after block with a carry between them."""
    snap = random_snapshot(seed, P=200, N=N, G=30, L=5, case="mixed", value_scale="big")
    _walkable_groups(snap.groups)
    return Case(f"big_values_N{N}", snap, np.arange(snap.pods.n, dtype=np.uint32),
                dict(cached=0, fitmask=1, n_blocks=-(-N // BLOCK)))


# ---- representative-class borders ----
BORDER_N = 2 * BLOCK


def class_border(n_classes: int, seed: int = 21) -> Case:
    """n_classes representative classes; group 0 is the last of them (id n_classes - 1: pods' classes come first,
    then the groups').  Group 0 is in case A and its need on the cpu lane is exactly the cluster's total, which only
    the last node of block 1 reaches.  Queue: a pod of group 0 that passes the check but fits no node (so nothing
    changes), an ungrouped pod assumed onto node 1 (block 0 goes stale for every class), the group's pod again:
    the total is one short now, so the verdict flips to NOT_ENOUGH.  With 32 classes the group's class is 31, whose
    summary rows (62, 63) are the last the assume invalidates."""
    L = 5
    filler = n_classes - 1                          # pod classes besides group 0's own
    snap = random_snapshot(seed, P=filler + 3, N=BORDER_N, G=1, L=L, case="A")
    nt = snap.nodes
    _clean_nodes(nt, 4000, np.where(np.arange(BORDER_N) % 3 == 0, 4000, 3000))
    total = int((nt.alloc[0] - nt.requested[0]).sum())
    gt = snap.groups
    gt.flags[:] = S.GROUP_HAS_POD | S.GROUP_HAS_MINRES
    gt.min_member[0], gt.scheduled[0], gt.matched[0] = 1, 0, 0
    gt.min_res[:, 0] = 0
    gt.min_res[0, 0] = total
    gt.min_res_present[0] = 0
    gt.rep_sel[0], gt.rep_tol[0] = 0, 1000      # a class of its own, after every pod class
    pt = snap.pods
    pt.req[:] = 0
    pt.req_present[:] = 0
    pt.flags[:] = 0
    pt.sel_mask[:] = 0
    pt.tol_mask[:] = np.arange(pt.n) % filler     # `filler` pod classes
    pt.gid[:] = S.GID_NONE
    pt.gid[0] = 0
    pt.req[0, 0] = 1 << 40                          # passes the check, fits no node
    pt.req[0, 1] = 1                                # ungrouped: first fit is node 1 (node 0 is full)
    q = np.array([0, 1, 0], np.uint32)
    reg = dict(n_rep=n_classes, fitmask=int(n_classes <= MAX_CLASSES), cached=int(n_classes <= MAX_CLASSES),
               n_blocks=2)
    return Case(f"classes_{n_classes}", snap, q, reg, dict(total=total, group_class=n_classes - 1))


def many_classes_with_affinity(seed: int = 91) -> Case:
    """More than 32 representative classes and affinity classes: no fit mask, so the walk evaluates checkFit and
    the affinity bit of every node inline."""
    snap = random_snapshot(seed, P=300, N=2600, G=40, L=5, case="mixed", aff=3)
    rng = np.random.default_rng(seed)
    snap.pods.tol_mask[:] = rng.integers(0, 1 << 20, snap.pods.n).astype(np.uint64) | np.uint64(0xF)
    _walkable_groups(snap.groups)
    return Case("many_classes_affinity", snap, np.arange(snap.pods.n, dtype=np.uint32),
                dict(fitmask=0, cached=0, n_blocks=3))


# ---- the dead-node skip ----
DEAD_N = 3000
SURVIVOR = 700
SMALL_CPU = 100


def dead_node(variant: str, seed: int = 31) -> Case:
    """Block 0 leaves every node 50 cpu, below the table's smallest cpu request (100), except node 700, which
    leaves exactly 100 ("edge") or 99 ("below").  Blocks 1 and 2 have room.  Ungrouped pods of 500 / 2000 cpu go
    there; the last pod asks for 100.  "edge": node 700 is never dead, the skip never fires (lo 0) and the last pod
    lands there.  "below": block 0 is all dead, lo is 1024 and the last pod lands in block 1.  "negative": as
    "edge", plus a pod (not queued) with a negative cpu request, so the walk cannot skip at all (monotone 0, lo 0)."""
    P = 40
    snap = random_snapshot(seed, P=P, N=DEAD_N, G=4, L=5)
    nt = snap.nodes
    i = np.arange(DEAD_N)
    left0 = np.where(i < BLOCK, 50, 64000)
    left0[SURVIVOR] = SMALL_CPU - (variant == "below")
    _clean_nodes(nt, np.where(i < BLOCK, 4000, 64000), np.where(i < BLOCK, 4000, 64000) - left0)
    pt = snap.pods
    pt.gid[:] = S.GID_NONE
    pt.flags[:] = 0
    pt.req[0] = np.where(np.arange(P) % 2 == 0, 500, 2000)
    pt.req[0, P - 2] = SMALL_CPU
    pt.req[1] = np.minimum(pt.req[1], 1 << 30)
    pt.req[3] = 0
    if variant == "negative":
        pt.req[0, P - 1] = -SMALL_CPU
    pt.req_present[:] = 0                           # no scalar request keeps the last pod off node 700
    q = np.array([p for p in range(P - 2)] + ([P - 1] if variant != "negative" else []) + [P - 2], np.uint32)
    reg = dict(monotone=int(variant != "negative"), lo=BLOCK if variant == "below" else 0, cached=1, n_blocks=3)
    return Case(f"dead_{variant}", snap, q, reg, dict(variant=variant, last_node=SURVIVOR if variant != "below" else None))


# ---- findMaxPG buckets ----
def bucket_keys(G: int):
    """t0 < t1 < t3: t0 in bucket 1 and t1 in bucket 2, both at an offset past the first 32 groups of their
    bucket, t3 the table's last group (last bucket)."""
    size, _ = buckets(G)
    return size + 40, 2 * size + 50, G - 1


def bucket_border(G: int, case: str, seed: int = 41) -> Case:
    """Three groups tie at the maximum `finished`: t0 (scheduled >= min_member), t1 (scheduled 0) one bucket
    later, which replaces it (core.go:729-731), and t3 in the last bucket, which does not (first index wins).
    Case B: they tie at 5000 (t1 and t3 have matched 5 of min_member 1) and t1's class fits no node, so every pod
    of another group whose check runs against t1 is NOT_ENOUGH.  Case A: every group has matched 0 and they tie at
    0; the walk's assumes then make new maxima in whichever bucket a pod lands.  No other group starts above the
    tie."""
    snap = random_snapshot(seed, P=2000, N=300, G=G, L=5, case=case)
    gt = snap.groups
    rng = np.random.default_rng(seed)
    _walkable_groups(gt)
    gt.flags &= ~np.uint8(S.GROUP_HAS_POD)          # a group enters findMaxPG when its first pod arrives
    gt.scheduled[:] = 0
    t0, t1, t3 = bucket_keys(G)
    if case == "B":
        gt.min_member[:] = rng.integers(2, 9, G)
        gt.matched[:] = np.minimum(gt.matched, gt.min_member - 1)      # finished < 1000 < 5000
        gt.min_member[[t0, t1, t3]] = 1
        gt.scheduled[t0], gt.matched[t0] = 5, 0     # (0 + 5) * 1000 / 1
        gt.matched[[t1, t3]] = 5                    # 5 * 1000 / 1
        gt.rep_sel[t1] = UNFIT_SEL
    else:
        gt.min_member[t0], gt.scheduled[t0] = 2, 2  # min_member - scheduled == 0: finished 0
    gt.flags[[t0, t1, t3]] |= S.GROUP_HAS_POD | S.GROUP_HAS_MINRES
    pt = snap.pods
    pt.gid[:8] = [t0, t1, t3, t1, t3, t0, t3, t1]   # the key groups' pods come first
    size, nb = buckets(G)
    reg = dict(bucket_size=size, n_buckets=nb)
    return Case(f"buckets_{case}_G{G}", snap, np.arange(pt.n, dtype=np.uint32), reg,
                dict(keys=(t0, t1, t3), tie=5000 if case == "B" else 0))


# ---- the findMaxPG panic ----
def panic(variant: str) -> Case:
    """The README scenario plus group 2 with min_member 0, scheduled 3 and no pod yet.  Its pod arrives at queue
    position 3 with OCC_NOREFS (PreFilter stops before findMaxPG, but the group now has its pod), and the next step
    that reaches findMaxPG divides by zero: position 4.  "quiet": the pods after it are ungrouped, so no step
    reaches findMaxPG again.  "zero": scheduled 0, so min_member - scheduled == 0 and finished is 0: no divide."""
    base = S.readme_scenario()
    L = base.lanes
    gt = S.GroupTable.empty(3, L)
    gt.min_member[:] = [5, 5, 0]
    gt.scheduled[2] = 0 if variant == "zero" else 3
    gt.creation_ns[:] = base.groups.creation_ns[0]
    gt.name_rank[:] = [0, 1, 2]
    pt = S.PodTable.empty(11, L)
    pt.gid[:] = [0] * 5 + [1] * 5 + [2]
    pt.req[0, :] = 1000
    pt.ts_ns[:] = base.pods.ts_ns[0] + np.arange(11) * 1000
    pt.flags[10] = S.POD_OCC_NOREFS
    if variant == "quiet":
        pt.gid[5:10] = S.GID_NONE
    snap = S.Snapshot(base.nodes, pt, gt, f"panic_{variant}")
    q = np.array([0, 5, 1, 10, 2, 6, 3, 7, 4, 8, 9], np.uint32)
    if variant == "quiet":
        q = np.array([0, 1, 2, 10, 5, 6, 7], np.uint32)
    return Case(f"panic_{variant}", snap, q, dict(n_buckets=1, bucket_size=32, n_blocks=1), dict(variant=variant),
                priority=False, panic_at=4 if variant == "panic" else None)


# ---- small edges of first-fit bs_replay ----
def small(N: int, G: int = 30, seed: int = 51) -> Case:
    snap = random_snapshot(seed + N, P=120, N=max(N, 1), G=G, L=5, case="mixed")
    if N == 0:
        snap.nodes = snap.nodes.take(np.zeros(0, np.int64))
    _walkable_groups(snap.groups)
    size, nb = buckets(G)
    return Case(f"small_N{N}_G{G}", snap, np.random.default_rng(seed).permutation(snap.pods.n).astype(np.uint32),
                dict(n_blocks=-(-N // BLOCK), cached=int(N > 0), bucket_size=size, n_buckets=nb), priority=False)


@functools.cache
def cases() -> dict:
    out = [cache_limit(CACHE_N, "A"), cache_limit(CACHE_N, "B"), cache_limit(CACHE_N + 1, "A"),
           big_values(2600), big_values(5000),
           class_border(31), class_border(32), class_border(33), many_classes_with_affinity(),
           dead_node("edge"), dead_node("below"), dead_node("negative"),
           *(bucket_border(G, c) for G in (32768, 32769, 100000) for c in ("A", "B")),
           panic("panic"), panic("quiet"), panic("zero"),
           small(0), small(50, G=0), *(small(n) for n in (1, 1023, 1024, 1025, 2047, 2049))]
    return {c.name: c for c in out}
