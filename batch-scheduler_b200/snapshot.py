"""Snapshot tables (SoA, int64 lanes) and the synthetic generators of the benchmark configs.

The three tables are the flattened inputs of the reference hot path:
  * NodeTable  <- frameworkHandler.SnapshotSharedLister().NodeInfos().List()
                  (pkg/scheduler/core/core.go:597), fields read at core.go:647-668;
  * PodTable   <- the pods handed to PreFilter / Permit / Compare (core.go:88,268,368);
  * GroupTable <- cache.PGStatusCache.PGStatusMap (pkg/scheduler/cache/cache.go:45-67)
                  plus PodGroup Spec/Status (pkg/apis/podgroup/v1/types.go:79-130).
Lane order: 0 MilliCPU, 1 Memory, 2 EphemeralStorage, 3 AllowedPodNumber, 4.. scalars.
Lane-major layout: arr[d, i] == value of lane d for row i (C-contiguous [lanes][rows]).
"""
from __future__ import annotations

from dataclasses import dataclass, field
import numpy as np

FIXED_LANES = 4
MAX_LANES = 16
LANE_CPU, LANE_MEM, LANE_EPH, LANE_PODS = 0, 1, 2, 3

NODE_NIL, NODE_NO_NODE, NODE_UNSCHEDULABLE, NODE_TAINTS_ERR = 0x01, 0x02, 0x04, 0x08
POD_PERMITTED_RECENTLY, POD_OCC_NOREFS, POD_OCC_MISMATCH, POD_LISTER_MISS = 0x01, 0x02, 0x04, 0x08
GROUP_SCHEDULED, GROUP_HAS_POD, GROUP_HAS_MINRES, GROUP_DENIED = 0x01, 0x02, 0x04, 0x08
GID_NONE, GID_MISSING = -1, -2
AFF_NONE = 0xFFFFFFFF

PF_PASS, PF_NOT_FOUND, PF_DENIED, PF_OCC_NOREFS, PF_OCCUPIED, PF_NOT_ENOUGH = range(6)
ADMIT, WAIT, UNSCHEDULABLE = 0, 1, 2

GiB = 1 << 30
MiB = 1 << 20


def _c(a, dt):
    return np.ascontiguousarray(a, dtype=dt)


@dataclass
class NodeTable:
    alloc: np.ndarray          # int64 [L, N]
    requested: np.ndarray      # int64 [L, N]
    pod_count: np.ndarray      # int32 [N]
    alloc_present: np.ndarray  # uint32 [N]
    req_present: np.ndarray    # uint32 [N]
    label_mask: np.ndarray     # uint64 [N]
    taint_mask: np.ndarray     # uint64 [N]
    flags: np.ndarray          # uint8 [N]

    def __post_init__(self):
        self.alloc = _c(self.alloc, np.int64)
        self.requested = _c(self.requested, np.int64)
        self.pod_count = _c(self.pod_count, np.int32)
        self.alloc_present = _c(self.alloc_present, np.uint32)
        self.req_present = _c(self.req_present, np.uint32)
        self.label_mask = _c(self.label_mask, np.uint64)
        self.taint_mask = _c(self.taint_mask, np.uint64)
        self.flags = _c(self.flags, np.uint8)
        assert self.alloc.shape == self.requested.shape and self.alloc.ndim == 2

    @property
    def n(self):
        return self.alloc.shape[1]

    @property
    def lanes(self):
        return self.alloc.shape[0]

    @staticmethod
    def empty(n, lanes):
        z = lambda dt: np.zeros(n, dt)
        return NodeTable(np.zeros((lanes, n), np.int64), np.zeros((lanes, n), np.int64), z(np.int32),
                         z(np.uint32), z(np.uint32), z(np.uint64), z(np.uint64), z(np.uint8))

    def copy(self):
        return NodeTable(*(getattr(self, f).copy() for f in self.__dataclass_fields__))

    def take(self, idx):
        idx = np.asarray(idx)
        return NodeTable(self.alloc[:, idx], self.requested[:, idx], self.pod_count[idx], self.alloc_present[idx],
                         self.req_present[idx], self.label_mask[idx], self.taint_mask[idx], self.flags[idx])


@dataclass
class PodTable:
    req: np.ndarray          # int64 [L, P]
    req_present: np.ndarray  # uint32 [P]
    gid: np.ndarray          # int32 [P]
    sel_mask: np.ndarray     # uint64 [P]
    tol_mask: np.ndarray     # uint64 [P]
    priority: np.ndarray     # int32 [P]
    ts_ns: np.ndarray        # int64 [P]
    flags: np.ndarray        # uint8 [P]
    aff_class: np.ndarray = None   # uint32 [P] row of Snapshot.aff_bits, AFF_NONE = no affinity constraint; None = all NONE

    def __post_init__(self):
        if self.aff_class is not None:
            self.aff_class = _c(self.aff_class, np.uint32)
        self.req = _c(self.req, np.int64)
        self.req_present = _c(self.req_present, np.uint32)
        self.gid = _c(self.gid, np.int32)
        self.sel_mask = _c(self.sel_mask, np.uint64)
        self.tol_mask = _c(self.tol_mask, np.uint64)
        self.priority = _c(self.priority, np.int32)
        self.ts_ns = _c(self.ts_ns, np.int64)
        self.flags = _c(self.flags, np.uint8)
        assert self.req.ndim == 2

    @property
    def n(self):
        return self.req.shape[1]

    @property
    def lanes(self):
        return self.req.shape[0]

    @staticmethod
    def empty(n, lanes):
        z = lambda dt: np.zeros(n, dt)
        return PodTable(np.zeros((lanes, n), np.int64), z(np.uint32), np.full(n, GID_NONE, np.int32),
                        z(np.uint64), z(np.uint64), z(np.int32), z(np.int64), z(np.uint8))

    def copy(self):
        return PodTable(*(None if getattr(self, f) is None else getattr(self, f).copy() for f in self.__dataclass_fields__))

    def take(self, idx):
        idx = np.asarray(idx)
        return PodTable(self.req[:, idx], self.req_present[idx], self.gid[idx], self.sel_mask[idx],
                        self.tol_mask[idx], self.priority[idx], self.ts_ns[idx], self.flags[idx],
                        None if self.aff_class is None else self.aff_class[idx])


@dataclass
class GroupTable:
    min_member: np.ndarray       # uint32 [G]
    scheduled: np.ndarray        # uint32 [G]
    matched: np.ndarray          # uint32 [G]
    flags: np.ndarray            # uint8 [G]
    min_res: np.ndarray          # int64 [L, G]
    min_res_present: np.ndarray  # uint32 [G]
    rep_sel: np.ndarray          # uint64 [G]
    rep_tol: np.ndarray          # uint64 [G]
    creation_ns: np.ndarray      # int64 [G]
    name_rank: np.ndarray        # uint32 [G]
    rep_aff: np.ndarray = None   # uint32 [G] affinity class of pgs.Pod (AFF_NONE = none); None = all NONE

    def __post_init__(self):
        if self.rep_aff is not None:
            self.rep_aff = _c(self.rep_aff, np.uint32)
        self.min_member = _c(self.min_member, np.uint32)
        self.scheduled = _c(self.scheduled, np.uint32)
        self.matched = _c(self.matched, np.uint32)
        self.flags = _c(self.flags, np.uint8)
        self.min_res = _c(self.min_res, np.int64)
        self.min_res_present = _c(self.min_res_present, np.uint32)
        self.rep_sel = _c(self.rep_sel, np.uint64)
        self.rep_tol = _c(self.rep_tol, np.uint64)
        self.creation_ns = _c(self.creation_ns, np.int64)
        self.name_rank = _c(self.name_rank, np.uint32)
        assert self.min_res.ndim == 2

    @property
    def n(self):
        return self.min_res.shape[1]

    @property
    def lanes(self):
        return self.min_res.shape[0]

    @staticmethod
    def empty(n, lanes):
        z = lambda dt: np.zeros(n, dt)
        return GroupTable(z(np.uint32), z(np.uint32), z(np.uint32), z(np.uint8),
                          np.zeros((lanes, n), np.int64), z(np.uint32), z(np.uint64), z(np.uint64),
                          z(np.int64), z(np.uint32))

    def copy(self):
        return GroupTable(*(None if getattr(self, f) is None else getattr(self, f).copy() for f in self.__dataclass_fields__))

    def take(self, idx):
        idx = np.asarray(idx)
        return GroupTable(self.min_member[idx], self.scheduled[idx], self.matched[idx], self.flags[idx],
                          self.min_res[:, idx], self.min_res_present[idx], self.rep_sel[idx], self.rep_tol[idx],
                          self.creation_ns[idx], self.name_rank[idx],
                          None if self.rep_aff is None else self.rep_aff[idx])


BOUND_GROUP_LOCKED = 0x01   # the bound pod's PodGroup Status.Phase is Scheduled or Running


@dataclass
class BoundPodTable:
    """The pods already bound to the snapshot's nodes (NodeInfo.Pods()): what preemption may evict."""
    node: np.ndarray         # uint32 [V] node index
    req: np.ndarray          # int64 [L, V] the containers' Requests (lane 3 ignored)
    req_present: np.ndarray  # uint32 [V] scalar keys, a subset of the node's req_present
    gid: np.ndarray          # int32 [V] group index, GID_NONE (no group label) or GID_MISSING
    priority: np.ndarray     # int32 [V]
    start_ns: np.ndarray     # int64 [V] Status.StartTime
    flags: np.ndarray        # uint8 [V] BOUND_*

    def __post_init__(self):
        self.node = _c(self.node, np.uint32)
        self.req = _c(self.req, np.int64)
        self.req_present = _c(self.req_present, np.uint32)
        self.gid = _c(self.gid, np.int32)
        self.priority = _c(self.priority, np.int32)
        self.start_ns = _c(self.start_ns, np.int64)
        self.flags = _c(self.flags, np.uint8)
        assert self.req.ndim == 2 and self.req.shape[1] == len(self.node)

    @property
    def n(self):
        return self.req.shape[1]

    @property
    def lanes(self):
        return self.req.shape[0]

    @staticmethod
    def empty(n, lanes):
        z = lambda dt: np.zeros(n, dt)
        return BoundPodTable(z(np.uint32), np.zeros((lanes, n), np.int64), z(np.uint32), z(np.int32), z(np.int32),
                             z(np.int64), z(np.uint8))

    def copy(self):
        return BoundPodTable(*(getattr(self, f).copy() for f in self.__dataclass_fields__))


@dataclass
class Snapshot:
    nodes: NodeTable
    pods: PodTable
    groups: GroupTable
    name: str = ""
    meta: dict = field(default_factory=dict)
    aff_bits: np.ndarray = None   # uint32 [n_aff, ceil(N/32)]: (affinity class, node) predicate bits, or None

    @property
    def lanes(self):
        return self.nodes.lanes

    @property
    def pairs(self):
        return self.pods.n * self.nodes.n

    def copy(self):
        return Snapshot(self.nodes.copy(), self.pods.copy(), self.groups.copy(), self.name,
                        dict(self.meta), None if self.aff_bits is None else self.aff_bits.copy())

    def resolve_groups(self) -> "Snapshot":
        """Applies fillOccupiedObj's first-pod capture (core.go:486-493) on the host, over the WHOLE
        pod table: for every group the first pod (table order) that reaches fillOccupiedObj becomes
        pgs.Pod (HAS_POD + rep masks) and, if Spec.MinResources is nil, supplies it (HAS_MINRES).
        The engine does the same on device for the pods it sees; sharding must resolve first, because
        findMaxPG (core.go:701) reads this state for groups whose pods live on another rank."""
        s = self.copy()
        pt, gt = s.pods, s.groups
        G = gt.n
        if G == 0 or pt.n == 0:
            return s
        gid = pt.gid
        ok = (gid >= 0) & (gid < G) & ((pt.flags & POD_PERMITTED_RECENTLY) == 0)
        ok &= (gt.flags[np.clip(gid, 0, G - 1)] & GROUP_DENIED) == 0
        first = np.full(G, pt.n, np.int64)
        idx = np.nonzero(ok)[0]
        np.minimum.at(first, gid[idx], idx)
        has = first < pt.n
        fp = np.where(has, first, 0)
        take_pod = has & ((gt.flags & GROUP_HAS_POD) == 0)
        take_res = has & ((gt.flags & GROUP_HAS_MINRES) == 0)
        gt.rep_sel = np.where(take_pod, pt.sel_mask[fp], gt.rep_sel)
        gt.rep_tol = np.where(take_pod, pt.tol_mask[fp], gt.rep_tol)
        if pt.aff_class is not None:
            base = gt.rep_aff if gt.rep_aff is not None else np.full(G, AFF_NONE, np.uint32)
            gt.rep_aff = np.where(take_pod, pt.aff_class[fp], base).astype(np.uint32)
        pres = pt.req_present[fp] & ~np.uint32(0xF)
        for d in range(gt.lanes):
            lane_present = np.ones(G, bool) if d < 4 else ((pres >> np.uint32(d)) & 1).astype(bool)
            gt.min_res[d] = np.where(take_res, np.where(lane_present, pt.req[d][fp], 0), gt.min_res[d])
        gt.min_res_present = np.where(take_res, pres, gt.min_res_present).astype(np.uint32)
        gt.flags = (gt.flags | np.where(take_pod, GROUP_HAS_POD, 0).astype(np.uint8)
                    | np.where(take_res, GROUP_HAS_MINRES, 0).astype(np.uint8))
        return s

    def shard_groups(self, rank: int, world: int) -> "Snapshot":
        """Rank-local snapshot: contiguous group range balanced by pod count (SURVEY §8e).

        The node table and the group table are replicated; only the pods of the
        rank's groups (and the ungrouped pods with index % world == rank) stay.
        Call on a snapshot that went through resolve_groups()."""
        P, G = self.pods.n, self.groups.n
        per_group = np.bincount(self.pods.gid[self.pods.gid >= 0], minlength=G)
        cum = np.concatenate([[0], np.cumsum(per_group)])
        total = cum[-1]
        bounds = [int(np.searchsorted(cum, total * r / world, side="left")) for r in range(world + 1)]
        bounds[0], bounds[-1] = 0, G
        g0, g1 = bounds[rank], bounds[rank + 1]
        gid = self.pods.gid
        keep = ((gid >= g0) & (gid < g1)) | ((gid < 0) & (np.arange(P) % world == rank))
        idx = np.nonzero(keep)[0]
        s = Snapshot(self.nodes, self.pods.take(idx), self.groups, f"{self.name}[{rank}/{world}]",
                     dict(self.meta), self.aff_bits)
        s.meta.update(group_range=(g0, g1), pod_index=idx)
        return s


def bound_pods(snap: Snapshot, seed: int, fill: float = 1.0, max_per_node: int = None,
               priorities=(-10, 0, 0, 5, 100, 1000), n_starts: int = 8, online: float = 0.3, missing: float = 0.03,
               locked: float = 0.2) -> BoundPodTable:
    """A bound-pod table consistent with the node table: node n gets round(fill * pod_count[n]) pods (at most
    max_per_node) whose lanes 0-2 split the node's requested amounts (the last pod takes the remainder) and whose scalar
    keys are a random subset of the node's req_present.  Priorities are drawn from `priorities`, start times from
    n_starts values (ties on purpose); a pod is online (no group label) with probability `online`, in a missing group
    with `missing`, else in a random group of the snapshot, locked (Scheduled / Running) with `locked`."""
    rng = np.random.default_rng(seed)
    nt, G, L = snap.nodes, snap.groups.n, snap.nodes.lanes
    k = np.round(np.clip(nt.pod_count.astype(np.int64), 0, None) * fill).astype(np.int64)
    if max_per_node is not None:
        k = np.minimum(k, max_per_node)
    node = np.repeat(np.arange(nt.n, dtype=np.int64), k)
    V = len(node)
    bt = BoundPodTable.empty(V, L)
    bt.node = node.astype(np.uint32)
    if V:
        last = np.cumsum(k)[k > 0] - 1   # the last row of each non-empty node
        w = rng.random(V) + 0.1
        wsum = np.bincount(node, weights=w, minlength=nt.n)
        for d in range(3):
            total = nt.requested[d][node]
            part = np.floor(total.astype(np.float64) * (w / wsum[node])).astype(np.int64)
            part[last] = 0
            part[last] = nt.requested[d][node[last]] - np.bincount(node, weights=part, minlength=nt.n)[node[last]].astype(np.int64)
            bt.req[d] = part
        pres = np.zeros(V, np.uint32)
        for d in range(4, L):
            has = ((nt.req_present[node] >> np.uint32(d)) & 1).astype(bool) & (rng.random(V) < 0.6)
            pres |= has.astype(np.uint32) << np.uint32(d)
            bt.req[d] = np.where(has, rng.integers(0, 4, V), 0)
        bt.req_present = pres
        bt.priority = rng.choice(np.asarray(priorities, np.int64), V).astype(np.int32)
        bt.start_ns = (1_600_000_000 * 10**9 + rng.integers(0, n_starts, V) * 10**9).astype(np.int64)
        u = rng.random(V)
        gid = rng.integers(0, G, V) if G else np.full(V, GID_NONE)
        gid = np.where(u < online, GID_NONE, np.where(u < online + missing, GID_MISSING, gid))
        bt.gid = gid.astype(np.int32)
        bt.flags = np.where((gid >= 0) & (rng.random(V) < locked), BOUND_GROUP_LOCKED, 0).astype(np.uint8)
    return bt


DEFAULT_MILLI_CPU_REQUEST = 100                 # GetNonzeroRequests: a container without a cpu request
DEFAULT_MEMORY_REQUEST = 200 * 1024 * 1024      # ... and without a memory request
NONZERO_MAX = 1 << 56


def nonzero_requests(snap: Snapshot, seed: int, explicit_zero: float = 0.1, unset_on_node: int = 4):
    """Seeded non-zero request columns (BS_OUT_PRIORITY) for a table without containers: (node [2, N], pod [2, P])
    int64, row 0 cpu (millicores), row 1 memory (bytes).  The stand-in: a pod is one container whose Requests are its
    req lanes 0-1; a zero there is an absent key (counted as 100 m / 200 MiB) except with probability `explicit_zero`,
    where it is an explicit zero and stays 0.  A node's column is its requested lanes 0-1 plus 0..unset_on_node pods
    without any request (each counted at both defaults).  Values are clipped into [0, 2^56]."""
    rng = np.random.default_rng(seed)
    nt, pt = snap.nodes, snap.pods
    pod = np.zeros((2, pt.n), np.int64)
    for row, lane, dflt in ((0, LANE_CPU, DEFAULT_MILLI_CPU_REQUEST), (1, LANE_MEM, DEFAULT_MEMORY_REQUEST)):
        r = pt.req[lane].astype(np.int64)
        absent = (r == 0) & (rng.random(pt.n) >= explicit_zero)
        pod[row] = np.where(absent, dflt, r)
    unset = rng.integers(0, unset_on_node + 1, nt.n).astype(np.int64)
    node = np.stack([nt.requested[LANE_CPU].astype(np.int64) + unset * DEFAULT_MILLI_CPU_REQUEST,
                     nt.requested[LANE_MEM].astype(np.int64) + unset * DEFAULT_MEMORY_REQUEST])
    return np.clip(node, 0, NONZERO_MAX), np.clip(pod, 0, NONZERO_MAX)


# ----------------------------------------------------------------------------
# splitmix64 stream (vectorised): value i of the stream with seed s is
# mix(s + (i+1)*0x9E3779B97F4A7C15).
class SplitMix64:
    GOLDEN = np.uint64(0x9E3779B97F4A7C15)

    def __init__(self, seed: int):
        self.seed = np.uint64(seed & 0xFFFFFFFFFFFFFFFF)
        self.pos = 0

    def u64(self, n: int) -> np.ndarray:
        with np.errstate(over="ignore"):
            i = np.arange(self.pos + 1, self.pos + n + 1, dtype=np.uint64)
            z = self.seed + i * self.GOLDEN
            z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
            z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
            z = z ^ (z >> np.uint64(31))
        self.pos += n
        return z

    def below(self, n: int, bound: int) -> np.ndarray:
        return (self.u64(n) % np.uint64(bound)).astype(np.int64)

    def choice(self, n: int, values) -> np.ndarray:
        v = np.asarray(values)
        return v[self.below(n, len(v))]

    def uniform(self, n: int) -> np.ndarray:
        return (self.u64(n) >> np.uint64(11)).astype(np.float64) / float(1 << 53)

    def bernoulli_bits(self, n: int, bits: int, prob: float) -> np.ndarray:
        out = np.zeros(n, np.uint64)
        for b in range(bits):
            out |= (self.uniform(n) < prob).astype(np.uint64) << np.uint64(b)
        return out


def _synth(seed: int, G: int, group_sizes: np.ndarray, min_member: np.ndarray, N: int, S: int,
           name: str, shuffle_pods: bool = False, shard: int = 0) -> Snapshot:
    """Synthetic snapshot per SURVEY.md §8(d).  Nodes come from their own stream (seed), groups
    and pods from a second stream that also depends on `shard`: rank r of a weak-scaling run
    gets the same (replicated) node table and its own groups/pods."""
    rng = SplitMix64(seed)
    L = FIXED_LANES + S
    # ---- nodes ----
    nt = NodeTable.empty(N, L)
    nt.alloc[LANE_CPU] = rng.choice(N, [16, 32, 64, 96, 128]) * 1000
    mem = rng.choice(N, [64, 128, 256, 512, 1024]).astype(np.int64) * GiB
    mem -= rng.below(N, 2048) * MiB + (rng.below(N, 512) * 2 + 1)  # odd byte offset: exercises float32 rounding
    nt.alloc[LANE_MEM] = mem
    nt.alloc[LANE_EPH] = (100 + rng.below(N, 1900)) * GiB
    nt.alloc[LANE_PODS] = 110
    for s in range(S):
        d = FIXED_LANES + s
        vals = [0, 4, 8] if s == 0 else [0, 0, 0, 2, 16]
        a = rng.choice(N, vals).astype(np.int64)
        nt.alloc[d] = a
        has = a > 0
        nt.alloc_present |= (has.astype(np.uint32) << np.uint32(d))
        # requested map holds the key on 90% of the nodes that expose the resource (quirk Q2)
        rp = has & (rng.uniform(N) < 0.9)
        nt.req_present |= (rp.astype(np.uint32) << np.uint32(d))
        used = np.floor(a * rng.uniform(N) * 0.9).astype(np.int64)
        nt.requested[d] = np.where(rp, used, 0)
    fr = rng.uniform(N) * 0.9
    nt.requested[LANE_CPU] = (np.floor(nt.alloc[LANE_CPU] * fr / 10) * 10).astype(np.int64)
    fr = rng.uniform(N) * 0.9
    nt.requested[LANE_MEM] = (np.floor(nt.alloc[LANE_MEM] * fr / MiB)).astype(np.int64) * MiB
    fr = rng.uniform(N) * 0.9
    nt.requested[LANE_EPH] = (np.floor(nt.alloc[LANE_EPH] * fr / MiB)).astype(np.int64) * MiB
    nt.pod_count = rng.below(N, 61).astype(np.int32)
    nt.flags = np.where(rng.uniform(N) < 0.01, NODE_UNSCHEDULABLE, 0).astype(np.uint8)
    nt.label_mask = rng.bernoulli_bits(N, 8, 0.2)
    nt.taint_mask = rng.bernoulli_bits(N, 4, 0.05)

    # ---- groups (pods homogeneous within a group) ----
    rng = SplitMix64((seed ^ 0x6A09E667F3BCC908) + 0x1000 * shard)
    gt = GroupTable.empty(G, L)
    g_cpu = rng.choice(G, [250, 500, 1000, 2000, 4000, 8000]).astype(np.int64)
    g_mem = (rng.choice(G, [0.25, 1, 4, 16, 32]) * GiB).astype(np.int64)
    g_eph = rng.choice(G, [0, 1, 10]).astype(np.int64) * GiB
    g_sc = np.zeros((S, G), np.int64)
    for s in range(S):
        vals = [0, 0, 0, 1, 2, 4, 8] if s == 0 else [0, 0, 0, 0, 0, 1, 2]
        g_sc[s] = rng.choice(G, vals)
    # 20% of the groups pin one label bit; 30% tolerate every taint
    sel_pick = rng.below(G, 8)
    g_sel = np.where(rng.uniform(G) < 0.2, np.uint64(1) << sel_pick.astype(np.uint64), np.uint64(0)).astype(np.uint64)
    g_tol = np.where(rng.uniform(G) < 0.3, np.uint64(0xF), np.uint64(0)).astype(np.uint64)
    gt.min_member = min_member.astype(np.uint32)
    gt.min_res[LANE_CPU], gt.min_res[LANE_MEM], gt.min_res[LANE_EPH] = g_cpu, g_mem, g_eph
    for s in range(S):
        d = FIXED_LANES + s
        gt.min_res[d] = g_sc[s]
        gt.min_res_present |= ((g_sc[s] > 0).astype(np.uint32) << np.uint32(d))
    carried = rng.uniform(G) < 0.05
    m_carry = np.where(min_member > 1, 1 + rng.below(G, 1 << 30) % np.maximum(min_member - 1, 1), 0)
    gt.matched = np.where(carried, m_carry, 0).astype(np.uint32)
    denied = rng.uniform(G) < 0.02
    gt.flags = (GROUP_HAS_POD | GROUP_HAS_MINRES | np.where(denied, GROUP_DENIED, 0)).astype(np.uint8)
    gt.rep_sel, gt.rep_tol = g_sel, g_tol
    t0 = 1_600_000_000 * 1_000_000_000
    gt.creation_ns = t0 + rng.below(G, 3600) * 1_000_000_000
    gt.name_rank = np.arange(G, dtype=np.uint32)  # names pg-%07d sort like their index
    g_prio = rng.below(G, 10).astype(np.int32)

    # ---- pods ----
    P = int(group_sizes.sum())
    gid = np.repeat(np.arange(G, dtype=np.int32), group_sizes)
    pt = PodTable.empty(P, L)
    pt.gid = gid
    pt.req[LANE_CPU], pt.req[LANE_MEM], pt.req[LANE_EPH] = g_cpu[gid], g_mem[gid], g_eph[gid]
    for s in range(S):
        d = FIXED_LANES + s
        pt.req[d] = g_sc[s][gid]
        pt.req_present |= ((g_sc[s][gid] > 0).astype(np.uint32) << np.uint32(d))
    pt.sel_mask, pt.tol_mask = g_sel[gid], g_tol[gid]
    pt.priority = g_prio[gid]
    pt.ts_ns = t0 + 3600 * 1_000_000_000 + rng.below(P, 600_000_000) * 1000
    if shuffle_pods:
        perm = np.argsort(rng.u64(P), kind="stable")
        pt = pt.take(perm)
    snap = Snapshot(nt, pt, gt, name, dict(seed=seed, S=S))
    return snap


def config(cfg: int, scale: float = 1.0, shard: int = 0) -> Snapshot:
    """BASELINE.json configs #2..#5 (SURVEY.md §8(d)); `scale` shrinks P, N, G together for tests;
    `shard` selects the rank-local groups/pods of a weak-scaling run (nodes are replicated)."""
    seed = 0xB2000000 + cfg
    sc = lambda x: max(1, int(round(x * scale)))
    if cfg == 2:
        G, N = sc(1000), sc(1000)
        return _synth(seed, G, np.full(G, 8), np.full(G, 8), N, 1, "cfg2: 1k groups x 8 pods, 1k nodes, 5 lanes",
                      shard=shard)
    if cfg == 3:
        G, N = sc(10000), sc(10000)
        rng = SplitMix64(seed ^ 0x5555)
        mm = 1 + rng.below(G, 16)
        return _synth(seed, G, np.full(G, 16), mm, N, 1, "cfg3: 10k groups x 16 pods, 10k nodes, minMember 1-16",
                      shard=shard)
    if cfg == 4:
        G, N = sc(50000), sc(10000)
        rng = SplitMix64(seed ^ 0x5555)
        sizes = 1 + rng.below(G, 3)
        # exactly 100k pods at scale 1: fix the drift on the last groups
        target = sc(100000)
        diff = int(sizes.sum()) - target
        i = 0
        while diff != 0 and i < 10 * G:
            j = i % G
            if diff > 0 and sizes[j] > 1:
                sizes[j] -= 1; diff -= 1
            elif diff < 0 and sizes[j] < 3:
                sizes[j] += 1; diff += 1
            i += 1
        return _synth(seed, G, sizes, sizes.copy(), N, 1,
                      "cfg4: 100k pods / 10k nodes, 50k groups, priority-sorted queue", shuffle_pods=True,
                      shard=shard)
    if cfg == 5:
        G, N = sc(62500), sc(50000)
        return _synth(seed, G, np.full(G, 16), np.full(G, 16), N, 5,
                      "cfg5: 1M pods / 50k nodes, 62.5k groups, 9 lanes", shard=shard)
    raise ValueError(f"unknown config {cfg}")


def readme_scenario() -> Snapshot:
    """BASELINE config #1: README.md:76-188 — one 8-cpu node with 900m / 140Mi requested,
    two PodGroups (minMember 5) of five 1-cpu pods each."""
    L = 4
    nt = NodeTable.empty(1, L)
    nt.alloc[LANE_CPU, 0] = 8000
    nt.alloc[LANE_MEM, 0] = 16 * GiB
    nt.alloc[LANE_EPH, 0] = 100 * GiB
    nt.alloc[LANE_PODS, 0] = 110
    nt.requested[LANE_CPU, 0] = 900
    nt.requested[LANE_MEM, 0] = 140 * MiB
    nt.pod_count[0] = 4
    gt = GroupTable.empty(2, L)
    gt.min_member[:] = 5
    t0 = 1_600_000_000 * 1_000_000_000
    gt.creation_ns[:] = [t0, t0]
    gt.name_rank[:] = [0, 1]  # "group1" < "group2"
    pt = PodTable.empty(10, L)
    pt.gid[:] = [0] * 5 + [1] * 5
    pt.req[LANE_CPU, :] = 1000
    pt.ts_ns[:] = t0 + np.arange(10) * 1000
    return Snapshot(nt, pt, gt, "cfg1: README resource-race example")


def core_test_cases():
    """pkg/scheduler/core/core_test.go:27-115 as tables: one node (10 cpu, 10 nvidia-gpu,
    20 tencentip, 100 pods) already holding the pod; three pods -> expected [True, False, False].
    Lanes: 4 = alpha.kubernetes.io/nvidia-gpu, 5 = tencent.cr/tencentip."""
    L = 6
    nt = NodeTable.empty(1, L)
    nt.alloc[LANE_CPU, 0] = 10000
    nt.alloc[LANE_PODS, 0] = 100
    nt.alloc[4, 0] = 10
    nt.alloc[5, 0] = 20
    nt.alloc_present[0] = (1 << 4) | (1 << 5)
    # nodeIf.AddPod(&pod): requested = the pod's Requests (cpu 1, gpu 1, ip 1); len(Pods()) = 1
    nt.requested[LANE_CPU, 0] = 1000
    nt.requested[4, 0] = 1
    nt.requested[5, 0] = 1
    nt.req_present[0] = (1 << 4) | (1 << 5)
    nt.pod_count[0] = 1
    pt = PodTable.empty(3, L)
    pt.req[LANE_CPU, :] = 1000
    pt.req[4, :] = [1, 101, 1]
    pt.req[5, :] = [1, 1, 101]
    pt.req_present[:] = (1 << 4) | (1 << 5)
    gt = GroupTable.empty(0, L)
    expected = [True, False, False]
    expected_left = dict(cpu=9000, mem=0, eph=0, pods=99, gpu=9, ip=19)
    return Snapshot(nt, pt, gt, "core_test.go:27-115"), expected, expected_left
