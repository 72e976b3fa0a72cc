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
BOUND_PDB_VIOLATING = 0x02  # the bound pod violates a PodDisruptionBudget (filterPodsWithPDBViolation)


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
               locked: float = 0.2, violating: float = 0.0) -> BoundPodTable:
    """A bound-pod table consistent with the node table: node n gets round(fill * pod_count[n]) pods (at most
    max_per_node) whose lanes 0-2 split the node's requested amounts (the last pod takes the remainder) and whose scalar
    keys are a random subset of the node's req_present.  Priorities are drawn from `priorities`, start times from
    n_starts values (ties on purpose); a pod is online (no group label) with probability `online`, in a missing group
    with `missing`, else in a random group of the snapshot, locked (Scheduled / Running) with `locked`.  A pod violates
    a PodDisruptionBudget with probability `violating`, drawn after everything else and only when it is > 0, so that a
    seed gives the same table with the default as without the parameter."""
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
        if violating > 0:
            bt.flags |= np.where(rng.random(V) < violating, BOUND_PDB_VIOLATING, 0).astype(np.uint8)
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


PREF_NONE = 0xFFFFFFFF   # BS_PREF_NONE


def node_preferences(snap: Snapshot, seed: int, n_bits: int = 6, tainted: float = 0.3, tolerate: float = 0.4,
                     tolerate_all: float = 0.1, n_classes: int = 5, terms: int = 3, match: float = 0.3,
                     no_class: float = 0.3):
    """Seeded columns of the TaintToleration and preferred NodeAffinity priorities for a table without objects:
    (prefer_taints [N] uint64, pref_weights [n_classes, N] int32, prefer_tol [P] uint64, pref_class [P] uint32).
    A share `tainted` of the nodes carries a random non-empty subset of n_bits PreferNoSchedule taints; a pod tolerates
    each bit with probability `tolerate`, or every bit with `tolerate_all`.  A class is `terms` preferred terms of
    weight 1..100, each matching a node with probability `match`; a pod has no class (PREF_NONE) with `no_class`."""
    rng = np.random.default_rng(seed)
    N, P = snap.nodes.n, snap.pods.n
    bits = rng.random((N, n_bits)) < 0.5
    bits[np.arange(N), rng.integers(0, max(n_bits, 1), N)] = True   # non-empty
    taint_bits = (bits & (rng.random(N) < tainted)[:, None]) if n_bits else np.zeros((N, 0), bool)
    weights_of_bits = np.uint64(1) << np.arange(n_bits, dtype=np.uint64)
    prefer_taints = (taint_bits.astype(np.uint64) * weights_of_bits).sum(axis=1, dtype=np.uint64)
    tol_bits = (rng.random((P, n_bits)) < tolerate) | (rng.random(P) < tolerate_all)[:, None]
    prefer_tol = (tol_bits.astype(np.uint64) * weights_of_bits).sum(axis=1, dtype=np.uint64)
    pref_weights = np.zeros((n_classes, N), np.int64)
    for c in range(n_classes):
        for _ in range(terms):
            pref_weights[c] += np.where(rng.random(N) < match, int(rng.integers(1, 101)), 0)
    pref_class = rng.integers(0, max(n_classes, 1), P).astype(np.uint32)
    if n_classes == 0:
        pref_class[:] = PREF_NONE
    pref_class[rng.random(P) < no_class] = PREF_NONE
    return prefer_taints.astype(np.uint64), pref_weights.astype(np.int32), prefer_tol.astype(np.uint64), pref_class


IMAGE_NONE = 0xFFFFFFFF   # BS_IMAGE_NONE
AVOID_NONE = 0xFF         # BS_AVOID_NONE
MIB = 1 << 20


def node_locality(snap: Snapshot, seed: int, n_images: int = 16, n_classes: int = 8, max_ids: int = 5,
                  no_image: float = 0.2, n_controllers: int = 8, avoided: float = 0.1, controlled: float = 0.6):
    """Seeded columns of the ImageLocality and NodePreferAvoidPods priorities for a table without objects:
    (node, pods) with node = (image_size [I] int64, image_bits [I, ceil(N/32)] uint32, avoid_mask [N] uint64) and
    pods = (image_class [P] uint32, class_offset [C+1] uint32, class_images [nnz] uint32, avoid_bit [P] uint8).
    Sizes span 0 to 20 GiB; four names lie on every node at 23 MiB, 23 MiB + 1, 1000 MiB - 1 and 1000 MiB, so that
    sums land on and next to both thresholds; the others are reported by a share of the nodes drawn from
    {1 node, 5 %, 30 %, 70 %, all}.  A class lists 1..max_ids ids drawn with replacement (duplicates count twice); a
    pod has no class (IMAGE_NONE) with `no_image`.  A share `avoided` of the nodes lists 1-2 of n_controllers
    controllers, and a pod has a controller bit with `controlled`, else AVOID_NONE."""
    rng = np.random.default_rng(seed)
    N, P = snap.nodes.n, snap.pods.n
    W = (N + 31) // 32
    fixed = [23 * MIB, 23 * MIB + 1, 1000 * MIB - 1, 1000 * MIB]
    size = np.zeros(n_images, np.int64)
    size[:min(4, n_images)] = fixed[:min(4, n_images)]
    rest = max(n_images - 4, 0)
    size[4:] = np.where(rng.random(rest) < 0.15, 0, (rng.random(rest) ** 3 * (20 << 30)).astype(np.int64))
    present = np.zeros((n_images, N), bool)
    present[:4] = True
    for i in range(4, n_images):
        share = rng.choice([-1.0, 0.05, 0.3, 0.7, 1.0])
        present[i] = rng.random(N) < share if share >= 0 else np.arange(N) == rng.integers(0, max(N, 1))
    padded = np.zeros((n_images, W * 32), bool)
    padded[:, :N] = present
    bits = (padded.reshape(n_images, W, 32).astype(np.uint64) << np.arange(32, dtype=np.uint64)).sum(
        axis=2, dtype=np.uint64).astype(np.uint32)
    lens = rng.integers(1, max_ids + 1, n_classes)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint32)
    ids = rng.integers(0, max(n_images, 1), int(off[-1])).astype(np.uint32)
    if n_classes and lens[0] >= 2 and n_images:
        ids[1] = ids[0]   # a duplicate image within a class
    cls = rng.integers(0, max(n_classes, 1), P).astype(np.uint32)
    cls[(rng.random(P) < no_image) | (n_classes == 0)] = IMAGE_NONE
    ctrl = rng.integers(0, n_controllers, (N, 2))
    avoid = (np.uint64(1) << ctrl[:, 0].astype(np.uint64)) | np.where(
        rng.random(N) < 0.5, np.uint64(1) << ctrl[:, 1].astype(np.uint64), np.uint64(0))
    avoid = np.where(rng.random(N) < avoided, avoid, np.uint64(0)).astype(np.uint64)
    abit = np.where(rng.random(P) < controlled, rng.integers(0, n_controllers, P), AVOID_NONE).astype(np.uint8)
    return (size, bits, avoid), (cls, off, ids, abit)


SPREAD_NONE = 0xFFFFFFFF   # BS_SPREAD_NONE
ZONE_NONE = 0xFF           # BS_ZONE_NONE


def node_spread(snap: Snapshot, seed: int, n_zones: int = 4, unzoned: float = 0.2, n_classes: int = 6,
                occupied: float = 0.3, max_count: int = 6, no_class: float = 0.25):
    """Seeded columns of the SelectorSpread priority for a table without objects: (node, pods) with node = (zone [N]
    uint8, counts [n_classes, N] int32) and pods = spread_class [P] uint32.  A share `unzoned` of the nodes has no zone
    (ZONE_NONE), the rest lie in one of n_zones zones; a class counts 1..max_count matching pods on a share `occupied`
    of the nodes and 0 elsewhere; a pod has no class (SPREAD_NONE) with `no_class`."""
    rng = np.random.default_rng(seed)
    N, P = snap.nodes.n, snap.pods.n
    zone = rng.integers(0, max(n_zones, 1), N).astype(np.uint8)
    zone[(rng.random(N) < unzoned) | (n_zones == 0)] = ZONE_NONE
    counts = np.where(rng.random((n_classes, N)) < occupied, rng.integers(1, max_count + 1, (n_classes, N)), 0)
    cls = rng.integers(0, max(n_classes, 1), P).astype(np.uint32)
    cls[(rng.random(P) < no_class) | (n_classes == 0)] = SPREAD_NONE
    return (zone, counts.astype(np.int32)), cls


IPA_NONE = 0xFFFFFFFF    # BS_IPA_NONE
TOPO_NONE = 0xFFFFFFFF   # BS_TOPO_NONE


def interpod_classes(rng, n_classes: int, n_terms: int, max_entries: int, max_weight: int = 100,
                     hard: int = 1) -> tuple:
    """A seeded class table (class_offset [C + 1], term, own int32, match uint8): each class lists 1..max_entries
    distinct terms; own is a preferred affinity (+1..max_weight), a preferred anti-affinity (-1..-max_weight), a
    required affinity (+hard) or nothing (0), and match is 0 or 1, so both signs and both directions occur."""
    off, term, own, match = [0], [], [], []
    for _ in range(n_classes):
        k = int(rng.integers(1, min(max_entries, max(n_terms, 1)) + 1)) if n_terms else 0
        ts = rng.choice(n_terms, k, replace=False) if k else []
        for t in ts:
            kind = int(rng.integers(0, 4))
            w = int(rng.integers(1, max_weight + 1))
            term.append(int(t))
            own.append((w, -w, hard, 0)[kind])
            match.append(int(rng.integers(0, 2)))
        off.append(len(term))
    return (np.array(off, np.uint32), np.array(term, np.uint32), np.array(own, np.int32), np.array(match, np.uint8))


def node_interpod(snap: Snapshot, seed: int, n_zones: int = 8, rack_size: int = 16, unlabelled: float = 0.05,
                  n_terms: int = 24, n_bound: int = None, n_bclasses: int = 12, n_pclasses: int = 10,
                  max_entries: int = 6, no_class: float = 0.2, hard: int = 1):
    """Seeded columns of the InterPodAffinity priority for a table without objects: (node, pods) as Engine.upload_interpod
    takes them.  Three topology keys: a hostname-like key (one value per node), a zone-like key (n_zones values) and a
    rack-like key (one value per rack_size nodes); a share `unlabelled` of the nodes lacks the zone and the rack key.
    n_terms terms over the three keys; n_bound bound pods (default 4 per node) spread over the nodes, of n_bclasses
    classes; n_pclasses pod classes; a share `no_class` of the pods and of the bound pods has no class (IPA_NONE)."""
    rng = np.random.default_rng(seed)
    N, P = snap.nodes.n, snap.pods.n
    n_bound = 4 * N if n_bound is None else n_bound
    racks = max((N + rack_size - 1) // rack_size, 1)
    n_values = np.array([max(N, 1), max(n_zones, 1), racks], np.uint32)
    topo = np.stack([np.arange(N), rng.integers(0, max(n_zones, 1), N), np.arange(N) // rack_size]).astype(np.uint32)
    topo[1:, rng.random(N) < unlabelled] = TOPO_NONE
    term_key = rng.integers(0, 3, n_terms).astype(np.uint32)
    bound_node = rng.integers(0, max(N, 1), n_bound).astype(np.uint32)
    bound_class = rng.integers(0, max(n_bclasses, 1), n_bound).astype(np.uint32)
    bound_class[(rng.random(n_bound) < no_class) | (n_bclasses == 0)] = IPA_NONE
    bcl = interpod_classes(rng, n_bclasses, n_terms, max_entries, hard=hard)
    pod_class = rng.integers(0, max(n_pclasses, 1), P).astype(np.uint32)
    pod_class[(rng.random(P) < no_class) | (n_pclasses == 0)] = IPA_NONE
    pcl = interpod_classes(rng, n_pclasses, n_terms, max_entries, hard=0)
    return (n_values, topo, term_key, bound_node, bound_class, bcl), (pod_class, pcl)


IPF_NONE = 0xFFFFFFFF                           # BS_IPF_NONE
IPF_AFFINITY, IPF_ANTI, IPF_EXISTING = range(3)  # BS_IPF_* roles


def node_interpod_filter(snap: Snapshot, seed: int, n_zones: int = 8, unlabelled: float = 0.05,
                         one_per_host: float = 0.3, ps_affine: float = 0.2, ps_missing: float = 0.1,
                         siblings: int = 2, n_blockers: int = 16, blocked: float = 0.1, filler: int = 2,
                         self_affine: float = 0.4):
    """Seeded columns of the MatchInterPodAffinity filter for a table without objects: (node, pods) as
    Engine.upload_interpod_filter takes them.  Two topology keys: a hostname-like key (one value per node) and a
    zone-like key (n_zones values; a share `unlabelled` of the nodes lacks it).  Per gang:
    - a share one_per_host carries required anti-affinity on the hostname key against its own job label, with up to
      `siblings` of its pods already bound;
    - a share ps_affine needs the zone of its labelled "ps" pod (required affinity, the workers do not match it
      themselves); for a share ps_missing of those the ps pod is not bound, so no node passes;
    - a share self_affine needs the zone of its own job (required affinity the workers match themselves, self_match 1)
      with up to `siblings` of its pods bound: none bound, or bound only on nodes without the zone key, leaves the
      first-pod exception to let every node pass.
    n_blockers bound pods carry required anti-affinity on the zone key, each against a label that the pods of a share
    `blocked` of the gangs carry.  `filler` bound pods per node have no class.  Own generator: other draws keep their
    seeds."""
    rng = np.random.default_rng(seed)
    N, G = snap.nodes.n, snap.groups.n
    gid = snap.pods.gid
    n_values = np.array([max(N, 1), max(n_zones, 1)], np.uint32)
    topo = np.stack([np.arange(N), rng.integers(0, max(n_zones, 1), N)]).astype(np.uint32)
    topo[1, rng.random(N) < unlabelled] = TOPO_NONE
    term_key, bnode, bcls = [], [], []
    boff, bterm, bown, bmatch = [0], [], [], []

    def term(key):
        term_key.append(key)
        return len(term_key) - 1

    def bound(node, entries):   # one bound pod with a class of its own: entries (term, own, match)
        for t, o, m in entries:
            bterm.append(t); bown.append(o); bmatch.append(m)
        boff.append(len(bterm))
        bnode.append(node)
        bcls.append(len(boff) - 2)

    gang_entries = [[] for _ in range(G)]
    anti = rng.random(G) < one_per_host
    ps = (rng.random(G) < ps_affine) & ~anti
    missing = rng.random(G) < ps_missing
    selfaff = (rng.random(G) < self_affine) & ~anti & ~ps
    nsib = rng.integers(0, siblings + 1, G)
    for g in range(G):
        if anti[g]:
            t = term(0)
            gang_entries[g].append((t, IPF_ANTI))
            for _ in range(int(rng.integers(0, siblings + 1))):
                bound(int(rng.integers(0, max(N, 1))), [(t, 0, 1)])
        elif ps[g]:
            t = term(1)
            gang_entries[g].append((t, IPF_AFFINITY))
            if not missing[g]:
                bound(int(rng.integers(0, max(N, 1))), [(t, 0, 1)])
        elif selfaff[g]:
            t = term(1)
            gang_entries[g].append((t, IPF_AFFINITY))
            for _ in range(int(nsib[g]) if N else 0):
                bound(int(rng.integers(0, N)), [(t, 0, 1)])
    for _ in range(n_blockers if N else 0):
        w = term(1)
        bound(int(rng.integers(0, N)), [(w, 1, 0)])
        for g in np.flatnonzero(rng.random(G) < blocked):
            gang_entries[g].append((w, IPF_EXISTING))
    bnode += rng.integers(0, max(N, 1), filler * N).tolist()
    bcls += [IPF_NONE] * (filler * N)
    cls_of_gang = np.full(G, IPF_NONE, np.uint32)
    poff, pterm, prole, pself = [0], [], [], []
    for g in range(G):
        ent = gang_entries[g][:64]
        if not ent:
            continue
        cls_of_gang[g] = len(poff) - 1
        pterm += [t for t, _ in ent]
        prole += [r for _, r in ent]
        poff.append(len(pterm))
        pself.append(1 if selfaff[g] else 0)
    ok = (gid >= 0) & (gid < G)
    pod_class = np.where(ok, cls_of_gang[np.clip(gid, 0, max(G - 1, 0))] if G else IPF_NONE, IPF_NONE).astype(np.uint32)
    node = (n_values, topo, np.array(term_key, np.uint32), np.array(bnode, np.uint32), np.array(bcls, np.uint32),
            (np.array(boff, np.uint32), np.array(bterm, np.uint32), np.array(bown, np.int32), np.array(bmatch, np.uint8)))
    pods = (pod_class, (np.array(poff, np.uint32), np.array(pterm, np.uint32), np.array(prole, np.uint8),
                        np.array(pself, np.uint8)))
    return node, pods


def node_interpod_walk(snap: Snapshot, seed: int, pending_ps: float = 0.8, **kw):
    """node_interpod_filter's columns (same seed and keywords, same draws) plus a placed side consistent with them, as
    Engine.upload_interpod_placed takes it: (node, pods, placed).  A gang's pods own and match their hostname
    anti-affinity term, match their self-affine set and match the blockers' terms their filter class lists as EXISTING.
    For a share pending_ps of the parameter-server gangs, one pod of the table without a filter class becomes the
    pending parameter server: its placed class matches the gang's affinity term.  Own generator: other draws keep
    their seeds."""
    node, pods = node_interpod_filter(snap, seed, **kw)
    pod_class, (poff, pterm, prole, pself) = pods
    rng = np.random.default_rng(seed + 0x5EED)
    qoff, qterm, qown, qmatch = [0], [], [], []
    qcls_of = np.full(len(pself), IPF_NONE, np.uint32)
    ps_terms = []
    for c in range(len(pself)):
        ent = []
        for k in range(poff[c], poff[c + 1]):
            t, r = int(pterm[k]), int(prole[k])
            if r == IPF_ANTI:
                ent.append((t, 1, 1))
            elif r == IPF_EXISTING or (r == IPF_AFFINITY and pself[c]):
                ent.append((t, 0, 1))
            elif r == IPF_AFFINITY:
                ps_terms.append(t)
        if ent:
            qcls_of[c] = len(qoff) - 1
            for t, o, m in ent:
                qterm.append(t); qown.append(o); qmatch.append(m)
            qoff.append(len(qterm))
    placed_class = np.where(pod_class != IPF_NONE, qcls_of[np.minimum(pod_class, max(len(pself) - 1, 0))]
                            if len(pself) else IPF_NONE, IPF_NONE).astype(np.uint32)
    free = list(rng.permutation(np.flatnonzero(pod_class == IPF_NONE)))
    for t in sorted(set(ps_terms)):
        if rng.random() >= pending_ps or not free:
            continue
        placed_class[free.pop()] = len(qoff) - 1
        qterm.append(t); qown.append(0); qmatch.append(1)
        qoff.append(len(qterm))
    placed = (placed_class, (np.array(qoff, np.uint32), np.array(qterm, np.uint32), np.array(qown, np.int32),
                             np.array(qmatch, np.uint8)))
    return node, pods, placed


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
