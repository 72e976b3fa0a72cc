"""Designed rounds in which one lane decides every outcome, for every lane count L = 4..16.

The lane count picks the build of the prefix scans (lane bounds 4, 5, 6, 8, 9, 12, 16) and of bs_replay
(lane bounds 5, 9, 16), and the lane classes of the fit kernel.  Random snapshots put small values on every scalar
lane, so the top lane seldom decides a verdict.  Here every lane but one is generous and never decides anything; the
deciding lane is present on some nodes and absent on others, its residuals sit at, just above and just below the
pods' requests, and the groups' MinResources on it decide the cluster checks:

  case "A"      every group has matched == 0: each pod's own group at percent 1.0.  Group needs are the deciding
                lane's largest prefix (true), that plus 1 (false), a prefix late in the table (true), and, for the
                class of nodes where the lane is absent or negative, 0 (true only through absence) and 1 (false).
  case "B"      the max group has matched 2 of MinMember 4: every other pod against 2 x its MinResources plus the
                pod's request at percent 0.7 (float32 scaling); the MinResources put the split between passing and
                failing requests at the largest prefix, late in the table.
  case "mixed"  as B, but the max group's class holds only the nodes where the lane is absent or negative and its
                need on the lane is 0: a pod passes only through the prefixes that lack the key.

Values: in A the deciding lane and the fixed lanes are narrow (for L >= 10 the FIT_MAX_LN cap turns the top scalar
lanes wide, or the round takes the all-wide fallback); in "mixed" the deciding lane is wide (2^36 + small) next to
narrow fixed lanes; in B every fixed lane is wide, so the round takes the all-wide fallback.

L = 4 has no scalar lane: there the pods lane (3) decides and presence plays no part.
"""
from __future__ import annotations

import numpy as np

from randsnap import S

LANES = tuple(range(4, 17))
CASES = ("A", "B", "mixed")
LEVELS = (0, 1, 2, 3, 5, 8, 13, 21)       # residuals above the lane's base on the nodes that hold the key
WIDE_BASE = 1 << 36
CLS_ALL, CLS_LOW = 0x1, 0x2               # label bits: every node / the nodes whose deciding lane is absent or < 0
PRES, NEG, AONLY, RONLY, NONE = range(5)  # the deciding lane on a node: present >= 0, present < 0, alloc key only,
#                                           requested key only, neither key
I64_MIN = np.iinfo(np.int64).min


def deciding_lanes(L):
    """The top lane and the bottom scalar lane (one lane for L = 4 and 5)."""
    return sorted({L - 1, 4 if L > 4 else 3})


def combos():
    return [(L, d, case) for L in LANES for d in deciding_lanes(L) for case in CASES]


def _base(case):
    """(base, unit): the deciding lane's residuals are base + level x unit.  float32 holds 2^36 + k x 2^13 exactly,
    so the wide residuals keep their levels through int64(float32(alloc) * 1.0)."""
    return (WIDE_BASE, 1 << 13) if case == "mixed" else (0, 1)


def scale(a, pct):
    """int64(float32(alloc) * percent), element-wise."""
    return (np.asarray(a, np.int64).astype(np.float32) * np.float32(pct)).astype(np.int64)


def lane_terms(nt, d, sel, pct):
    """singleNodeResource's value of lane d per node for class (sel, 0) at pct: (terms[N], keyed[N], visited[N])."""
    vis = (nt.flags & 0x07) == 0
    ok = vis & ((nt.flags & S.NODE_TAINTS_ERR) == 0) & ((nt.label_mask & np.uint64(sel)) == np.uint64(sel)) & \
        (nt.taint_mask == 0)
    if d == 3:
        used = np.where(nt.requested[3] != 0, nt.requested[3], nt.pod_count.astype(np.int64))
        keyed = ok.copy()
    else:
        used = nt.requested[d]
        keyed = ok & (((nt.alloc_present & nt.req_present) >> np.uint32(d)) & np.uint32(1)).astype(bool)
    return np.where(keyed, scale(nt.alloc[d], pct) - used, 0), keyed, vis


def lane_prefix(nt, d, sel, pct):
    """The cluster walk's running sum of lane d (compareClusterResourceAndRequire, core.go:595-632): prefix[N],
    whether the key has been seen by then, visited[N]."""
    t, keyed, vis = lane_terms(nt, d, sel, pct)
    return np.cumsum(t), np.logical_or.accumulate(keyed), vis


def max_prefix(nt, d, sel, pct):
    pre, seen, vis = lane_prefix(nt, d, sel, pct)
    has = vis & seen
    return int(pre[has].max()) if has.any() else 0


def _nodes(L, d, N, rng, wide_fixed, base, unit):
    nt = S.NodeTable.empty(N, L)
    odd = lambda lo, n: lo + 2 * rng.integers(0, 1 << 16, n) + 1
    if wide_fixed:
        nt.alloc[0], nt.alloc[1], nt.alloc[2] = odd(1 << 30, N), odd(1 << 38, N), odd(1 << 40, N)
        nt.alloc[3] = (1 << 28) + 111
    else:
        nt.alloc[0], nt.alloc[1], nt.alloc[2], nt.alloc[3] = 64000, odd(1 << 36, N), 1 << 20, 110
    nt.requested[0] = rng.integers(0, 1000, N)
    nt.requested[1] = rng.integers(0, 1 << 30, N)
    nt.requested[2] = rng.integers(0, 1000, N)
    nt.pod_count = rng.integers(0, 50, N).astype(np.int32)
    for e in range(4, L):
        if e != d:
            nt.alloc[e] = (1 << 35) + 1001 if wide_fixed else 1000
            nt.requested[e] = rng.integers(0, 10, N)
            nt.alloc_present |= np.uint32(1 << e)
            nt.req_present |= np.uint32(1 << e)
    # the deciding lane
    kind = rng.choice(5, N, p=[0.6, 0.12, 0.1, 0.08, 0.1])
    kind[:16] = rng.choice([AONLY, RONLY, NONE], 16)            # the first prefixes of class LOW lack the key
    if d < 4:
        kind = np.where(kind == NEG, NEG, PRES)
    lvl = rng.choice(LEVELS, N)
    # requested one unit and alloc = residual + one unit: the terms at 0.7 stay about 0.7 x the residual
    nt.alloc[d] = np.where(kind == PRES, base + (lvl + 1) * unit, 1)
    nt.requested[d] = np.where(kind == PRES, unit, np.where(kind == NEG, 1 + rng.choice([1, 4], N), 9))
    if d >= 4:
        bit = np.uint32(1 << d)
        nt.alloc_present |= np.where(np.isin(kind, (PRES, NEG, AONLY)), bit, np.uint32(0)).astype(np.uint32)
        nt.req_present |= np.where(np.isin(kind, (PRES, NEG, RONLY)), bit, np.uint32(0)).astype(np.uint32)
    nt.label_mask = np.where(kind == PRES, CLS_ALL, CLS_ALL | CLS_LOW).astype(np.uint64)
    skip = rng.choice(np.arange(16, N), max(2, N // 50), replace=False)
    nt.flags[skip] = np.where(np.arange(len(skip)) % 2 == 0, S.NODE_NIL, S.NODE_UNSCHEDULABLE)
    return nt


EXACT, PLUS1, ZERO = range(3)


def _pods(L, d, P, G, rng, base, unit):
    pt = S.PodTable.empty(P, L)
    kind = rng.choice(3, P, p=[0.45, 0.35, 0.2])
    lvl = rng.choice(LEVELS, P)
    pt.req[0] = rng.integers(0, 100, P)
    pt.req[1] = rng.integers(0, 1 << 20, P)
    pt.req[3] = rng.integers(0, 2, P)
    # a third of the pods ask for some of the other scalar lanes: Filter's getLeftResource carries no scalar key,
    # so there a request other than 0 on any lane decides alone
    other = rng.random(P) < 1 / 3
    for e in range(4, L):
        if e != d:
            pt.req[e] = np.where(other, rng.integers(0, 6, P), 0)
            pt.req_present |= (rng.random(P) < 0.5).astype(np.uint32) << np.uint32(e)
    # exactly a node's residual, one above it, or 0 (the pods of class LOW: they fit only where the key is absent)
    pt.req[d] = np.where(kind == EXACT, base + lvl * unit, np.where(kind == PLUS1, base + lvl * unit + 1, 0))
    if d >= 4:
        pt.req_present |= np.uint32(1 << d)
    pt.sel_mask = np.where(kind == ZERO, CLS_LOW, CLS_ALL).astype(np.uint64)
    pt.gid = rng.integers(0, G, P).astype(np.int32)
    pt.gid[rng.random(P) < 0.05] = S.GID_NONE
    pt.priority = rng.choice([0, 0, 1, 7], P).astype(np.int32)
    pt.ts_ns = 1_700_000_000 * 10**9 + rng.permutation(P) * 1000
    return pt, kind


def _groups(L, d, G, rng):
    gt = S.GroupTable.empty(G, L)
    gt.min_member[:] = 1
    gt.flags[:] = S.GROUP_HAS_POD | S.GROUP_HAS_MINRES
    gt.min_res[0], gt.min_res[1] = 10, 1 << 10
    for e in range(4, L):
        if e != d:
            gt.min_res[e, 1:] = 1              # the max group's 0: Filter's case 3 stays with the deciding lane
            gt.min_res_present |= (rng.random(G) < 0.3).astype(np.uint32) << np.uint32(e)
    if d >= 4:
        gt.min_res_present |= np.uint32(1 << d)
    gt.rep_sel[:] = CLS_ALL
    gt.creation_ns = 1_600_000_000 * 10**9 + rng.integers(0, 5, G) * 10**9
    gt.name_rank = rng.permutation(G).astype(np.uint32)
    return gt


def lane_snapshot(L, case, deciding_lane, seed, N=2300, P=201, G=40):
    """A round of L lanes in which lane `deciding_lane` decides the fit, the Filter matrix and the cluster checks."""
    d = deciding_lane
    assert 3 <= d < L and case in CASES
    rng = np.random.default_rng([seed, L, d, CASES.index(case)])
    base, unit = _base(case)
    nt = _nodes(L, d, N, rng, case == "B", base, unit)
    pt, kind = _pods(L, d, P, G, rng, base, unit)
    gt = _groups(L, d, G, rng)
    if case == "A":
        pre, seen, vis = lane_prefix(nt, d, CLS_ALL, 1.0)
        has = np.flatnonzero(vis & seen)
        top = max_prefix(nt, d, CLS_ALL, 1.0)
        for g in range(1, G):
            mode = g % 6
            if mode == 0:
                need = top
            elif mode == 1:
                need = top + 1
            elif mode in (2, 3):                 # a prefix in the last third of the table
                need = int(pre[rng.choice(has[has >= 2 * N // 3])])
            else:                                 # class LOW: 0 is met only where the key is still absent
                gt.rep_sel[g] = CLS_LOW
                need = 0 if mode == 4 else 1
            gt.min_res[d, g] = need
        if d == 3:
            gt.min_res[3] = np.maximum(gt.min_res[3], 1)     # 0 on the pods lane reads as MinMember + 1
    else:
        gt.min_member[0], gt.matched[0] = 4, 2
        if case == "B":
            # 2 x MinResources + request <= the largest prefix at 0.7  <=>  request <= base + 5
            gt.min_res[d, 0] = (max_prefix(nt, d, CLS_ALL, 0.7) - (base + 5)) // 2
        else:
            gt.rep_sel[0] = CLS_LOW
            # the pods lane has no key to lack: the split sits at the class's largest prefix instead
            gt.min_res[d, 0] = 0 if d >= 4 else (max_prefix(nt, d, CLS_LOW, 0.7) - 5) // 2
    return S.Snapshot(nt, pt, gt, f"lanes{L}_d{d}_{case}_s{seed}")


def small_snapshot(L, case, deciding_lane, seed):
    """The same design at a size the pure-Python restatement walks in well under a second."""
    return lane_snapshot(L, case, deciding_lane, seed, N=70, P=37, G=12)


def lane_insensitive(snap, lane):
    """A copy in which `lane` no longer matters: its presence bit is cleared on pods and groups (a fixed lane: the
    pods' requests and the groups' MinResources on it become 0)."""
    s = snap.copy()
    if lane >= 4:
        s.pods.req_present &= np.uint32(~(1 << lane) & 0xFFFFFFFF)
        s.groups.min_res_present &= np.uint32(~(1 << lane) & 0xFFFFFFFF)
    else:
        s.pods.req[lane] = 0
        s.groups.min_res[lane] = 0
    s.name = snap.name + "_insensitive"
    return s


def neighbour(d, L):
    return d - 1 if d >= 5 else (d + 1 if d + 1 < L else d - 1)


def swap_node_lanes(snap, a, b):
    """A copy whose node table has lanes a and b exchanged (values and presence bits); pods and groups stay."""
    s = snap.copy()
    nt = s.nodes
    for col in (nt.alloc, nt.requested):
        col[[a, b]] = col[[b, a]]
    for m in ("alloc_present", "req_present"):
        v = getattr(nt, m)
        ba, bb = (v >> np.uint32(a)) & np.uint32(1), (v >> np.uint32(b)) & np.uint32(1)
        v &= np.uint32(~((1 << a) | (1 << b)) & 0xFFFFFFFF)
        v |= (ba << np.uint32(b)) | (bb << np.uint32(a))
    s.name = snap.name + f"_swap{a}{b}"
    return s


def cluster_needs(snap, d, sel, pct, n=48, seed=0):
    """Needs whose lane d sits at, just above and just below prefixes of class (sel, 0) at pct, plus 0 and 1; every
    other lane asks little.  Returns need[L, n] int64 and npres[n] uint32."""
    rng = np.random.default_rng([seed, d, sel, int(pct * 10)])
    nt = snap.nodes
    L = nt.lanes
    pre, seen, vis = lane_prefix(nt, d, sel, pct)
    has = np.flatnonzero(vis & seen)
    top = max_prefix(nt, d, sel, pct)
    need = np.zeros((L, n), np.int64)
    need[0], need[1], need[3] = 10, 1 << 10, 1
    npres = np.zeros(n, np.uint32)
    for j in range(n):
        m = j % 6
        if m == 0:
            v = top + (j // 6) % 2
        elif m in (1, 2) and len(has):
            v = int(pre[rng.choice(has)]) + (m == 2)
        elif m == 3:
            v = 0
        elif m == 4:
            v = 1
        else:
            v = int(pre[has[-1]]) - 1 if len(has) else -1
        need[d, j] = v
        if d >= 4:
            npres[j] = (1 << d) | (int(rng.integers(0, 1 << L)) & ~0xF & ((1 << L) - 1))
            for e in range(4, L):
                if e != d:
                    need[e, j] = 0 if (npres[j] >> e) & 1 else 7
    return need, npres


def cluster_answers(oracle, snap, need, npres, sel, pct):
    return np.array([oracle.compare_cluster(snap.nodes, sel, 0, need[:, j], int(npres[j]), pct)
                     for j in range(need.shape[1])])


def add_stray_bits(snap, seed):
    """A copy whose pod, node and group presence masks also carry bits 0..3 and bits of lanes >= L, which no lane
    reads."""
    s = snap.copy()
    L = s.lanes
    rng = np.random.default_rng(seed)
    stray = (0xFFFFFFFF & ~((1 << L) - 1)) | 0xF

    def bits(n):
        return (rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32) & np.uint32(stray))
    s.pods.req_present |= bits(s.pods.n)
    s.nodes.alloc_present |= bits(s.nodes.n)
    s.nodes.req_present |= bits(s.nodes.n)
    s.groups.min_res_present |= bits(s.groups.n)
    s.name = snap.name + "_stray"
    return s


def oracle_outputs(oracle, snap, d, need_lane=True):
    """Everything the deciding lane can change, from the oracle: PreFilter codes, fit bitmap, Filter bitmap,
    compare_cluster answers for both classes at both percents, and the replay walk in table order.  With
    need_lane=False the cluster needs do not carry lane d (as lane_insensitive does to the groups)."""
    r = oracle.round(snap, want_bitmap=True, want_sort=False, want_filter=True)
    ans = []
    for sel in (CLS_ALL, CLS_LOW):
        for pct in (1.0, 0.7):
            need, npres = cluster_needs(snap, d, sel, pct)
            if not need_lane:
                if d >= 4:
                    npres &= np.uint32(~(1 << d) & 0xFFFFFFFF)
                else:
                    need[d] = 0
            ans.append(cluster_answers(oracle, snap, need, npres, sel, pct))
    pf, node, ready, _ = oracle.replay(snap)
    return dict(prefilter=r.prefilter, fit=r.fit_bitmap, filter=r.filter_bitmap, cluster=np.concatenate(ans),
                replay=np.stack([pf.astype(np.int32), node, ready.astype(np.int32)]))


def changed_entries(a, b):
    """Per output: the number of entries (bits, for the bitmaps) that differ."""
    out = {}
    for k in a:
        if k in ("fit", "filter"):
            out[k] = int(np.unpackbits((a[k] ^ b[k]).view(np.uint8)).sum())
        else:
            out[k] = int((np.asarray(a[k]) != np.asarray(b[k])).sum())
    return out
