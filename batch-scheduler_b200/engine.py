"""Python host wrapper over the C ABI: one Engine = one bs_engine handle on one GPU."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from . import capi
from .snapshot import BoundPodTable, NodeTable, PodTable, GroupTable, Snapshot


@dataclass
class PreemptResult:
    """bs_preempt's outputs: per preemptor the chosen node (-1 none), its victims (bound-table indices, reprieve order:
    the BOUND_PDB_VIOLATING ones first) at victims[victim_offset[i]:victim_offset[i + 1]], and the number of candidate
    nodes."""
    node: np.ndarray           # int32 [n]
    n_victims: np.ndarray      # uint32 [n]
    n_candidates: np.ndarray   # uint32 [n]
    victim_offset: np.ndarray  # uint32 [n + 1]
    victims: np.ndarray        # uint32 [victims_total]

    def victims_of(self, i):
        return self.victims[self.victim_offset[i]:self.victim_offset[i + 1]].tolist()


@dataclass
class PreemptWalkResult(PreemptResult):
    """bs_preempt_walk's outputs: PreemptResult's fields for the walk, plus per preemptor its outcome (capi.WALK_*)
    and per bound row the list position whose step evicted it (-1 none)."""
    outcome: np.ndarray = None      # uint32 [n]
    evicted_by: np.ndarray = None   # int32 [V]


@dataclass
class RoundResult:
    prefilter: np.ndarray
    feasible_count: np.ndarray
    best_node: np.ndarray
    best_score: np.ndarray
    admit: np.ndarray
    admit_bitmap: np.ndarray
    new_denied: np.ndarray
    order: np.ndarray
    rank: np.ndarray
    max_group: int
    max_finished: int
    filter_code: np.ndarray = None


_TABLE_C = {
    NodeTable: (capi.NodeTableC, ("alloc", "requested", "pod_count", "alloc_present", "req_present", "label_mask",
                                  "taint_mask", "flags")),
    GroupTable: (capi.GroupTableC, ("min_member", "scheduled", "matched", "flags", "min_res", "min_res_present",
                                    "rep_sel", "rep_tol", "creation_ns", "name_rank", "rep_aff")),
    BoundPodTable: (capi.BoundTableC, ("node", "req", "req_present", "gid", "priority", "start_ns", "flags")),
    PodTable: (capi.PodTableC, ("req", "req_present", "gid", "sel_mask", "tol_mask", "priority", "ts_ns", "flags",
                                "aff_class")),
}


def _table_c(table):
    """The C struct of a table, for uploads and row updates alike: its columns in field order, alive for the call."""
    cls, cols = _TABLE_C[type(table)]
    return cls(table.n, table.lanes, *(capi.ptr(getattr(table, c)) for c in cols))


def _interpod_classes(cl, keep):
    """The bs_interpod_classes of (class_offset [C + 1], term, own int32, match uint8); `keep` holds its arrays."""
    off, term, own, match = cl
    a = [np.ascontiguousarray(off, dtype=np.uint32).reshape(-1), np.ascontiguousarray(term, dtype=np.uint32),
         np.ascontiguousarray(own, dtype=np.int32), np.ascontiguousarray(match, dtype=np.uint8)]
    keep += a
    return capi.InterpodClassesC(max(len(a[0]) - 1, 0), *(capi.ptr(x) for x in a))


class Engine:
    def __init__(self, n_lanes: int, device: int = 0, fit_bitmap: bool = True, score: bool = False,
                 filter: bool = False, topk: int = 0, reasons: bool = False, priority_k: int = 0):
        """topk > 0 also keeps each pod's `topk` best fitting nodes and their scores (BS_OUT_TOPK, read with
        topk_rows); it cannot be combined with score=True, whose matrix holds them already.  reasons=True also counts,
        per pod, the nodes that reject it for each reason (BS_OUT_REASONS, read with reason_rows).  priority_k > 0 also
        keeps each pod's priority_k best fitting nodes under kube-scheduler's resource priorities (BS_OUT_PRIORITY, read
        with priority_rows; needs upload_nonzero before each round); with topk too, both lists have the same length."""
        if topk and priority_k and topk != priority_k:
            raise ValueError("topk and priority_k share the list length K: they must be equal")
        self.lib = capi.load()
        self.n_lanes = n_lanes
        self.topk = topk
        self.priority_k = priority_k
        self.out_flags = ((capi.OUT_FIT_BITMAP if fit_bitmap else 0) | (capi.OUT_SCORE if score else 0) |
                          (capi.OUT_FILTER if filter else 0) | (capi.OUT_TOPK if topk else 0) |
                          (capi.OUT_REASONS if reasons else 0) | (capi.OUT_PRIORITY if priority_k else 0))
        cfg = capi.Config(device, n_lanes, self.out_flags, topk or priority_k)
        h = C.c_void_p()
        rc = self.lib.bs_create(C.byref(cfg), C.byref(h))
        if rc != 0:
            raise capi.BsError(rc, self.lib.bs_strerror(rc).decode())
        self.h = h
        self.P = self.N = self.G = 0
        self._bound_rows = 0   # rows of the last bound-pod table uploaded (preempt_walk's evicted_by)
        self._res = None

    # -- lifecycle -------------------------------------------------------------------------
    def close(self):
        if getattr(self, "h", None):
            self.lib.bs_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != 0:
            msg = self.lib.bs_last_error(self.h).decode() or self.lib.bs_strerror(rc).decode()
            raise capi.BsError(rc, msg)

    # -- uploads ---------------------------------------------------------------------------
    def upload_nodes(self, nt: NodeTable):
        self._check(self.lib.bs_upload_nodes(self.h, C.byref(_table_c(nt))))
        self.N = nt.n

    def update_nodes(self, idx, rows: NodeTable):
        """Overwrites rows `idx` of the resident node table with `rows` (a compact NodeTable)."""
        idx = np.ascontiguousarray(idx, dtype=np.uint32)
        assert len(idx) == rows.n
        self._check(self.lib.bs_update_nodes(self.h, capi.ptr(idx), C.byref(_table_c(rows))))

    def upload_groups(self, gt: GroupTable):
        self._check(self.lib.bs_upload_groups(self.h, C.byref(_table_c(gt))))
        self.G = gt.n

    def update_groups(self, idx, rows: GroupTable):
        """Overwrites rows `idx` of the resident group table with `rows` (a compact GroupTable)."""
        idx = np.ascontiguousarray(idx, dtype=np.uint32)
        assert len(idx) == rows.n
        self._check(self.lib.bs_update_groups(self.h, capi.ptr(idx), C.byref(_table_c(rows))))

    def upload_pods(self, pt: PodTable):
        self._check(self.lib.bs_upload_pods(self.h, C.byref(_table_c(pt))))
        self.P = pt.n

    def upload_affinity(self, bits):
        """[n_classes, ceil(N/32)] uint32 host-evaluated (affinity class, node) predicate bits, or None to clear."""
        if bits is None:
            self._check(self.lib.bs_upload_affinity(self.h, 0, None))
            return
        bits = np.ascontiguousarray(bits, dtype=np.uint32)
        assert bits.ndim == 2 and bits.shape[1] == (self.N + 31) // 32
        self._check(self.lib.bs_upload_affinity(self.h, bits.shape[0], capi.ptr(bits)))

    def upload(self, snap: Snapshot):
        self.upload_nodes(snap.nodes)
        if getattr(snap, "aff_bits", None) is not None:
            self.upload_affinity(snap.aff_bits)
        self.upload_groups(snap.groups)
        self.upload_pods(snap.pods)

    def set_wait_time(self, default_ns: int, per_group_ns=None):
        if per_group_ns is None:
            self._check(self.lib.bs_set_wait_time(self.h, default_ns, None, 0))
        else:
            a = np.ascontiguousarray(per_group_ns, dtype=np.int64)
            self._check(self.lib.bs_set_wait_time(self.h, default_ns, capi.ptr(a), len(a)))

    # -- evaluation ------------------------------------------------------------------------
    def _alloc_results(self, out=None):
        P, G = self.P, self.G
        if out is not None:
            # numpy-style out=: refill a RoundResult of the same shape (a caller looping over rounds
            # avoids ~2.6 MB of fresh, page-faulting result arrays per call)
            if len(out.prefilter) != P or len(out.admit) != G or \
                    (out.filter_code is None) != (not (self.out_flags & capi.OUT_FILTER)):
                raise ValueError("out= does not match the uploaded tables")
            r = out
        else:
            r = self._new_results(P, G)
        c = capi.ResultsC(capi.ptr(r.prefilter), capi.ptr(r.feasible_count), capi.ptr(r.best_node),
                          capi.ptr(r.best_score), capi.ptr(r.admit), capi.ptr(r.admit_bitmap),
                          capi.ptr(r.new_denied), capi.ptr(r.order), capi.ptr(r.rank), -1, 0,
                          capi.ptr(r.filter_code) if r.filter_code is not None else None)
        return r, c

    def _new_results(self, P, G):
        r = RoundResult(np.zeros(P, np.uint8), np.zeros(P, np.uint32), np.zeros(P, np.int32), np.zeros(P, np.int64),
                        np.zeros(G, np.uint8), np.zeros((G + 31) // 32, np.uint32), np.zeros(G, np.uint8),
                        np.zeros(P, np.uint32), np.zeros(P, np.uint32), -1, 0,
                        np.zeros(P, np.uint8) if (self.out_flags & capi.OUT_FILTER) else None)
        return r

    def _view_results(self, c) -> RoundResult:
        """RoundResult whose arrays ARE the engine's pinned decision arena (bs_fetch_view): read-only, valid until
        the next evaluate / upload / update on this engine.  The numpy wrappers are cached per arena layout."""
        P, G = self.P, self.G
        key = (c.prefilter, c.feasible_count, c.best_node, c.best_score, c.admit, c.admit_bitmap, c.new_denied,
               c.order, c.rank, c.filter_code, P, G)
        if getattr(self, "_view_key", None) != key:
            def arr(addr, n, dt):
                dt = np.dtype(dt)
                if not addr or n == 0:
                    return np.zeros(0, dt)
                a = np.frombuffer((C.c_char * (n * dt.itemsize)).from_address(addr), dtype=dt)
                a.flags.writeable = False
                return a
            self._view = RoundResult(arr(c.prefilter, P, np.uint8), arr(c.feasible_count, P, np.uint32),
                                     arr(c.best_node, P, np.int32), arr(c.best_score, P, np.int64),
                                     arr(c.admit, G, np.uint8), arr(c.admit_bitmap, (G + 31) // 32, np.uint32),
                                     arr(c.new_denied, G, np.uint8), arr(c.order, P, np.uint32), arr(c.rank, P, np.uint32),
                                     -1, 0, arr(c.filter_code, P, np.uint8) if c.filter_code else None)
            self._view_key = key
        self._view.max_group, self._view.max_finished = int(c.max_group), int(c.max_finished)
        return self._view

    def evaluate(self, out=None, view=False) -> RoundResult:
        """One round.  view=True returns the decision vectors in place (zero-copy views of the engine's pinned arena,
        read-only, overwritten by the next round) instead of copies."""
        if view:
            c = capi.ResultsC()
            self._check(self.lib.bs_evaluate_view(self.h, C.byref(c)))
            return self._view_results(c)
        r, c = self._alloc_results(out)
        self._check(self.lib.bs_evaluate(self.h, C.byref(c)))
        r.max_group, r.max_finished = int(c.max_group), int(c.max_finished)
        return r

    def evaluate_async(self):
        self._check(self.lib.bs_evaluate_async(self.h))

    def sync(self):
        self._check(self.lib.bs_sync(self.h))

    def fetch(self, out=None, view=False) -> RoundResult:
        if view:
            c = capi.ResultsC()
            self._check(self.lib.bs_fetch_view(self.h, C.byref(c)))
            return self._view_results(c)
        r, c = self._alloc_results(out)
        self._check(self.lib.bs_fetch(self.h, C.byref(c)))
        r.max_group, r.max_finished = int(c.max_group), int(c.max_finished)
        return r

    def fit_rows(self, pod0=0, n=None) -> np.ndarray:
        n = self.P - pod0 if n is None else n
        W = (self.N + 31) // 32
        out = np.zeros((n, W), np.uint32)
        self._check(self.lib.bs_fetch_fit_rows(self.h, pod0, n, capi.ptr(out)))
        return out

    def filter_rows(self, pod0=0, n=None) -> np.ndarray:
        n = self.P - pod0 if n is None else n
        W = (self.N + 31) // 32
        out = np.zeros((n, W), np.uint32)
        self._check(self.lib.bs_fetch_filter_rows(self.h, pod0, n, capi.ptr(out)))
        return out

    def filter(self, pod: int, node: int):
        st = capi.StatusC()
        self._check(self.lib.bs_filter(self.h, pod, node, C.byref(st)))
        return st.code, st.reason, st.group

    def score_rows(self, pod0=0, n=None) -> np.ndarray:
        n = self.P - pod0 if n is None else n
        out = np.zeros((n, self.N), np.int64)
        self._check(self.lib.bs_fetch_score_rows(self.h, pod0, n, capi.ptr(out)))
        return out

    def topk_rows(self, pod0=0, n=None):
        """(nodes [n, K] int32, scores [n, K] int64): each pod's fitting nodes by score descending, then node index
        ascending; min(K, feasible_count) entries, padded with node -1 and score INT64_MIN."""
        n = self.P - pod0 if n is None else n
        nodes = np.zeros((n, self.topk), np.int32)
        scores = np.zeros((n, self.topk), np.int64)
        self._check(self.lib.bs_fetch_topk_rows(self.h, pod0, n, capi.ptr(nodes), capi.ptr(scores)))
        return nodes, scores

    def reason_rows(self, pod0=0, n=None) -> np.ndarray:
        """[n, 4 + L] uint32: bin b of row p = the nodes that reject pod pod0 + p for reason b (capi.REASON_*)."""
        n = self.P - pod0 if n is None else n
        out = np.zeros((n, 4 + self.n_lanes), np.uint32)
        self._check(self.lib.bs_fetch_reason_rows(self.h, pod0, n, capi.ptr(out)))
        return out

    # -- resource priorities (BS_OUT_PRIORITY) -------------------------------------------------
    def set_score_weights(self, least: int = 1, most: int = 0, balanced: int = 1):
        """Weights of LeastAllocated, MostAllocated and BalancedAllocation for the next rounds (default 1, 0, 1)."""
        self._check(self.lib.bs_set_score_weights(self.h, least, most, balanced))

    def set_ratio_priority(self, weight: int, shape, lane_weights, absent_weight: int = 0):
        """kube-scheduler's RequestedToCapacityRatio priority, added to the priority score with `weight` (0 = off).
        shape: (utilization, score) pairs in engine units (both 0..100, utilization strictly ascending); lane_weights:
        one weight per lane (lane 3 must be 0); absent_weight: the weights of resources no node has.  Read by the next
        rounds' priority lists and by replay(priority=True)."""
        pts = np.asarray(shape, dtype=np.int64).reshape(-1, 2)
        lw = np.asarray(lane_weights, dtype=np.int64).reshape(-1)
        if (pts < 0).any() or (pts > 0xFFFFFFFF).any() or (lw < 0).any() or (lw > 0xFFFFFFFF).any():
            raise ValueError("shape points and lane weights are unsigned 32-bit values")
        util = np.ascontiguousarray(pts[:, 0], dtype=np.uint32)
        score = np.ascontiguousarray(pts[:, 1], dtype=np.uint32)
        lw = np.ascontiguousarray(lw, dtype=np.uint32)
        self._check(self.lib.bs_set_ratio_priority(self.h, weight, len(util), capi.ptr(util), capi.ptr(score), len(lw),
                                                   capi.ptr(lw), absent_weight))

    def upload_nonzero(self, node=None, pods=None):
        """The non-zero request columns: node [2, N] and/or pods [2, P] int64 (row 0 cpu millicores, row 1 memory
        bytes).  Uploading nodes (or updating node rows) drops the node column, uploading pods the pod column."""
        if node is not None:
            a = np.ascontiguousarray(node, dtype=np.int64)
            self._check(self.lib.bs_upload_node_nonzero(self.h, a.shape[1] if a.ndim == 2 else 0, capi.ptr(a)))
        if pods is not None:
            a = np.ascontiguousarray(pods, dtype=np.int64)
            self._check(self.lib.bs_upload_pod_nonzero(self.h, a.shape[1] if a.ndim == 2 else 0, capi.ptr(a)))

    def set_node_priority_weights(self, taint_toleration: int = 0, node_affinity: int = 0):
        """Weights of kube-scheduler's TaintToleration and preferred NodeAffinity priorities in the priority score
        (0, 0 = off, the default; v1.17's default profile is 1, 1).  A non-zero weight needs upload_preferences before
        each round, and makes replay(priority=True) refuse to run."""
        self._check(self.lib.bs_set_node_priority_weights(self.h, taint_toleration, node_affinity))

    def upload_preferences(self, node=None, pods=None):
        """The columns of the two node priorities.  node = (prefer_taints [N] uint64, pref_weights [C, N] int32): bit b
        of prefer_taints is PreferNoSchedule taint b of the round's dictionary, pref_weights[c, n] the summed weights of
        class c's preferred terms that node n matches.  pods = (prefer_tol [P] uint64, pref_class [P] uint32): the bits
        each pod tolerates and its class (capi.PREF_NONE: no preferred terms).  Uploading nodes (or updating node rows)
        drops the node side, uploading pods the pod side."""
        if node is not None:
            taints = np.ascontiguousarray(node[0], dtype=np.uint64).reshape(-1)
            w = np.ascontiguousarray(node[1], dtype=np.int32)
            if w.ndim != 2 or w.shape[1] != len(taints):
                raise ValueError("pref_weights must be [classes, N] with N = len(prefer_taints)")
            self._check(self.lib.bs_upload_node_preferences(self.h, len(taints), capi.ptr(taints), w.shape[0],
                                                            capi.ptr(w)))
        if pods is not None:
            tol = np.ascontiguousarray(pods[0], dtype=np.uint64).reshape(-1)
            cls = np.ascontiguousarray(pods[1], dtype=np.uint32).reshape(-1)
            if len(tol) != len(cls):
                raise ValueError("prefer_tol and pref_class must have one entry per pod")
            self._check(self.lib.bs_upload_pod_preferences(self.h, len(tol), capi.ptr(tol), capi.ptr(cls)))

    def set_locality_weights(self, image_locality: int = 0, prefer_avoid_pods: int = 0):
        """Weights of kube-scheduler's ImageLocality and NodePreferAvoidPods priorities in the priority score and in
        replay(priority=True)'s node choice (0, 0 = off, the default; v1.17's default profile is 1, 10000).  A non-zero
        weight needs upload_locality before each round."""
        self._check(self.lib.bs_set_locality_weights(self.h, image_locality, prefer_avoid_pods))

    def upload_locality(self, node=None, pods=None):
        """The columns of the two locality priorities.  node = (image_size [I] int64, image_bits [I, ceil(N/32)]
        uint32, avoid_mask [N] uint64): the image dictionary's sizes in bytes, bit n%32 of word n/32 of row i set when
        node n reports name i, and bit b of avoid_mask when the node's preferAvoidPods annotation lists controller b.
        pods = (image_class [P] uint32, class_offset [C+1] uint32, class_images [nnz] uint32, avoid_bit [P] uint8):
        each pod's class (capi.IMAGE_NONE: none), the dictionary ids of each class (CSR), and each pod's controller bit
        (capi.AVOID_NONE: none).  Either image part or avoid part may be None when its weight is 0.  Uploading nodes
        (or updating node rows) drops the node side, uploading pods the pod side."""
        if node is not None:
            size, bits, avoid = node
            if size is not None:
                size = np.ascontiguousarray(size, dtype=np.int64).reshape(-1)
                bits = np.ascontiguousarray(bits, dtype=np.uint32).reshape(len(size), -1)
            if avoid is not None:
                avoid = np.ascontiguousarray(avoid, dtype=np.uint64).reshape(-1)
            n = len(avoid) if avoid is not None else self.N
            self._check(self.lib.bs_upload_node_locality(self.h, n, 0 if size is None else len(size), capi.ptr(size),
                                                         capi.ptr(bits), capi.ptr(avoid)))
        if pods is not None:
            cls, off, ids, abit = pods
            n_classes = 0
            if cls is not None:
                cls = np.ascontiguousarray(cls, dtype=np.uint32).reshape(-1)
                off = np.ascontiguousarray(off, dtype=np.uint32).reshape(-1)
                ids = np.ascontiguousarray(ids, dtype=np.uint32).reshape(-1)
                if len(off) < 1 or len(ids) < int(off[-1]):
                    raise ValueError("class_offset must have C+1 entries and class_images class_offset[C] of them")
                n_classes = len(off) - 1
            if abit is not None:
                abit = np.ascontiguousarray(abit, dtype=np.uint8).reshape(-1)
            if cls is not None and abit is not None and len(cls) != len(abit):
                raise ValueError("image_class and avoid_bit must have one entry per pod")
            n = len(cls) if cls is not None else len(abit) if abit is not None else self.P
            self._check(self.lib.bs_upload_pod_locality(self.h, n, capi.ptr(cls), n_classes, capi.ptr(off),
                                                        capi.ptr(ids), capi.ptr(abit)))

    def set_spread_weight(self, selector_spread: int = 0):
        """Weight of kube-scheduler's SelectorSpread priority in the priority score (0 = off, the default; v1.17's
        default profile is 1).  A non-zero weight needs upload_spread before each round, and makes
        replay(priority=True) refuse to run."""
        self._check(self.lib.bs_set_spread_weight(self.h, selector_spread))

    def upload_spread(self, node=None, pods=None, n_zones=None):
        """The columns of SelectorSpread.  node = (zone [N] uint8, counts [C, N] int32): each node's zone in the round's
        zone dictionary (capi.ZONE_NONE: no zone) and counts[c, n] the pods on node n that class c's selectors match.
        n_zones defaults to one more than the largest zone id.  pods = spread_class [P] uint32: each pod's class
        (capi.SPREAD_NONE: no selectors).  Uploading nodes (or updating node rows) drops the node side, uploading pods
        the pod side."""
        if node is not None:
            zone = np.ascontiguousarray(node[0], dtype=np.uint8).reshape(-1)
            counts = np.ascontiguousarray(node[1], dtype=np.int32)
            if counts.ndim != 2 or counts.shape[1] != len(zone):
                raise ValueError("counts must be [classes, N] with N = len(zone)")
            if n_zones is None:
                real = zone[zone != capi.ZONE_NONE]
                n_zones = int(real.max()) + 1 if len(real) else 0
            self._check(self.lib.bs_upload_node_spread(self.h, len(zone), n_zones, capi.ptr(zone), counts.shape[0],
                                                       capi.ptr(counts)))
        if pods is not None:
            cls = np.ascontiguousarray(pods, dtype=np.uint32).reshape(-1)
            self._check(self.lib.bs_upload_pod_spread(self.h, len(cls), capi.ptr(cls)))

    def set_interpod_weight(self, inter_pod_affinity: int = 0):
        """Weight of kube-scheduler's InterPodAffinity priority in the priority score (0 = off, the default; v1.17's
        default profile is 1).  A non-zero weight needs upload_interpod before each round, and makes
        replay(priority=True) refuse to run."""
        self._check(self.lib.bs_set_interpod_weight(self.h, inter_pod_affinity))

    def upload_interpod(self, node=None, pods=None):
        """The columns of InterPodAffinity (include/bsched.h bs_upload_node_interpod).  A class table is
        (class_offset [C + 1], term, own int32, match uint8).  node = (n_values [K], topo [K, N], term_key [T],
        bound_node [V], bound_class [V], classes): each key's value count, each node's value of each key
        (capi.TOPO_NONE: none), each term's key, the bound pods' nodes and classes (capi.IPA_NONE: none) and the bound
        classes.  pods = (pod_class [P], classes): each pod's class (capi.IPA_NONE: none) and the pod classes.  Uploading
        nodes (or updating node rows) drops the node side, uploading pods the pod side."""
        keep = []
        if node is not None:
            self._check(self.lib.bs_upload_node_interpod(self.h, C.byref(self._interpod_nodes(node, keep))))
        if pods is not None:
            pcls = np.ascontiguousarray(pods[0], dtype=np.uint32).reshape(-1)
            t = capi.InterpodPodsC(len(pcls), capi.ptr(pcls), _interpod_classes(pods[1], keep))
            self._check(self.lib.bs_upload_pod_interpod(self.h, C.byref(t)))

    def _interpod_nodes(self, node, keep):
        """The bs_interpod_nodes of upload_interpod's node tuple; `keep` holds its arrays for the call."""
        nv, topo, tkey, bnode, bcls, cl = node
        nv = np.ascontiguousarray(nv, dtype=np.uint32).reshape(-1)
        topo = (np.ascontiguousarray(topo, dtype=np.uint32).reshape(len(nv), -1) if len(nv)
                else np.zeros((0, self.N), np.uint32))
        tkey = np.ascontiguousarray(tkey, dtype=np.uint32).reshape(-1)
        bnode = np.ascontiguousarray(bnode, dtype=np.uint32).reshape(-1)
        bcls = np.ascontiguousarray(bcls, dtype=np.uint32).reshape(-1)
        if len(bnode) != len(bcls):
            raise ValueError("bound_node and bound_class must have one entry per bound pod")
        keep += [nv, topo, tkey, bnode, bcls]
        return capi.InterpodNodesC(topo.shape[1], len(nv), capi.ptr(nv), capi.ptr(topo), len(tkey), capi.ptr(tkey),
                                   len(bnode), capi.ptr(bnode), capi.ptr(bcls), _interpod_classes(cl, keep))

    def set_interpod_filter(self, on: bool = False):
        """Switch kube-scheduler's MatchInterPodAffinity filter (required pod affinity and anti-affinity) into every
        pod's fit set (off by default).  While it is on, each round needs upload_interpod_filter's two sides, replay
        needs upload_interpod_placed as well (it refuses to run without it), and preempt refuses to run."""
        self._check(self.lib.bs_set_interpod_filter(self.h, 1 if on else 0))

    def upload_interpod_filter(self, node=None, pods=None):
        """The columns of the MatchInterPodAffinity filter (include/bsched.h bs_upload_node_interpod_filter).  node: as
        upload_interpod's node side, with own 1 for a bound pod's required anti-affinity terms and match 1 for the terms
        it matches.  pods = (pod_class [P], (class_offset [C + 1], term, role uint8, self_match [C] uint8)): each pod's
        class (capi.IPF_NONE: none) and the class table with roles capi.IPF_AFFINITY / IPF_ANTI / IPF_EXISTING.
        Uploading nodes (or updating node rows) drops the node side, uploading pods the pod side."""
        if node is not None:
            keep = []
            self._check(self.lib.bs_upload_node_interpod_filter(self.h, C.byref(self._interpod_nodes(node, keep))))
        if pods is not None:
            pcls, (off, term, role, self_match) = pods
            a = [np.ascontiguousarray(pcls, dtype=np.uint32).reshape(-1),
                 np.ascontiguousarray(off, dtype=np.uint32).reshape(-1), np.ascontiguousarray(term, dtype=np.uint32),
                 np.ascontiguousarray(role, dtype=np.uint8), np.ascontiguousarray(self_match, dtype=np.uint8)]
            t = capi.InterpodFilterPodsC(len(a[0]), capi.ptr(a[0]), max(len(a[1]) - 1, 0), *(capi.ptr(x) for x in a[1:]))
            self._check(self.lib.bs_upload_pod_interpod_filter(self.h, C.byref(t)))

    def upload_interpod_placed(self, pod_class, classes):
        """The placed side of the MatchInterPodAffinity filter (include/bsched.h bs_upload_pod_interpod_placed): what
        each pending pod adds to presence once replay assumes it.  pod_class [P] (capi.IPF_NONE: nothing) and classes
        (class_offset [C + 1], term, own int32, match uint8) over the filter's dictionary, as a bound pod's class: own 1
        on the pod's required anti-affinity terms, match 1 on the terms it matches.  Uploading pods drops it."""
        keep = []
        pcls = np.ascontiguousarray(pod_class, dtype=np.uint32).reshape(-1)
        t = capi.InterpodPodsC(len(pcls), capi.ptr(pcls), _interpod_classes(classes, keep))
        self._check(self.lib.bs_upload_pod_interpod_placed(self.h, C.byref(t)))

    def fetch_interpod_reason_rows(self, pod0=0, n=None) -> np.ndarray:
        """[n, 3] uint32: the companion of reason_rows, the nodes that fail MatchInterPodAffinity after every other
        check, by step: existing pods' anti-affinity (E), the pod's affinity (A), the pod's anti-affinity (N)."""
        n = self.P - pod0 if n is None else n
        out = np.zeros((n, 3), np.uint32)
        self._check(self.lib.bs_fetch_interpod_reason_rows(self.h, pod0, n, capi.ptr(out)))
        return out

    def set_host_port_filter(self, on: bool = False):
        """Switch kube-scheduler's PodFitsHostPorts filter into every pod's fit set (off by default).  While it is on,
        each round needs upload_host_ports' two sides; replay applies it, and preempt and preempt_walk apply it once
        upload_bound_host_ports has given the bound pods' ports (they refuse to run without them)."""
        self._check(self.lib.bs_set_host_port_filter(self.h, 1 if on else 0))

    def upload_host_ports(self, node=None, pods=None):
        """The columns of the PodFitsHostPorts filter (include/bsched.h bs_upload_node_host_ports).  node = (entries,
        used): entries [K, 3] rows (ip id, protocol id, port), ip id capi.HOSTPORT_IP_ANY the wildcard "0.0.0.0", and
        used [N] uint64, bit k = the node uses entry k.  pods = want [P] uint64, bit k = the pod asks for entry k.
        Uploading nodes (or updating node rows) drops the node side, uploading pods the pod side."""
        if node is not None:
            entries, used = node
            ent = np.asarray(entries, dtype=np.int64).reshape(-1, 3)
            ip = np.ascontiguousarray(ent[:, 0], dtype=np.uint32)
            proto = np.ascontiguousarray(ent[:, 1], dtype=np.uint32)
            port = np.ascontiguousarray(np.clip(ent[:, 2], -1, 1 << 20), dtype=np.int32)
            used = np.ascontiguousarray(used, dtype=np.uint64).reshape(-1)
            t = capi.HostPortNodesC(len(used), len(ent), capi.ptr(ip), capi.ptr(proto), capi.ptr(port), capi.ptr(used))
            self._check(self.lib.bs_upload_node_host_ports(self.h, C.byref(t)))
        if pods is not None:
            want = np.ascontiguousarray(pods, dtype=np.uint64).reshape(-1)
            self._check(self.lib.bs_upload_pod_host_ports(self.h, len(want), capi.ptr(want)))

    def fetch_host_port_reason_rows(self, pod0=0, n=None) -> np.ndarray:
        """[n] uint32: the companion of reason_rows, the nodes past the guards that have a host-port conflict with the
        pod, whatever their other bins."""
        n = self.P - pod0 if n is None else n
        out = np.zeros(n, np.uint32)
        self._check(self.lib.bs_fetch_host_port_reason_rows(self.h, pod0, n, capi.ptr(out)))
        return out

    def priority_rows(self, pod0=0, n=None):
        """(nodes [n, K] int32, scores [n, K] int64): each pod's fitting nodes by priority score descending, then node
        index ascending; min(K, feasible_count) entries, padded with node -1 and score INT64_MIN."""
        n = self.P - pod0 if n is None else n
        nodes = np.zeros((n, self.priority_k), np.int32)
        scores = np.zeros((n, self.priority_k), np.int64)
        self._check(self.lib.bs_fetch_priority_rows(self.h, pod0, n, capi.ptr(nodes), capi.ptr(scores)))
        return nodes, scores

    def fit_error(self, counts, n_nodes: int, scalar_names=None) -> str:
        """The "0/N nodes are available: ..." message of one reason row (bs_format_fit_error)."""
        return format_fit_error(counts, self.n_lanes, n_nodes, scalar_names)

    def reasons_ms(self) -> float:
        """Milliseconds of the last round's reason-row stage (profiling on)."""
        ms, n = C.c_float(), C.c_uint32()
        self._check(self.lib.bs_kernel_ms(self.h, capi.K_REASONS, C.byref(ms), C.byref(n)))
        return float(ms.value)

    # -- standalone kernels ------------------------------------------------------------------
    def node_left(self, sel: int, tol: int, percent: float):
        left = np.zeros((self.n_lanes, self.N), np.int64)
        pres = np.zeros(self.N, np.uint32)
        self._check(self.lib.bs_node_left(self.h, sel, tol, C.c_float(percent), capi.ptr(left), capi.ptr(pres)))
        return left, pres

    def cluster_check(self, sel: int, tol: int, percent: float, need: np.ndarray, need_present: np.ndarray):
        need = np.ascontiguousarray(need, dtype=np.int64)  # [L, n]
        need_present = np.ascontiguousarray(need_present, dtype=np.uint32)
        n = need.shape[1]
        ok = np.zeros(n, np.uint8)
        self._check(self.lib.bs_cluster_check(self.h, sel, tol, C.c_float(percent), capi.ptr(need),
                                              capi.ptr(need_present), n, capi.ptr(ok)))
        return ok.astype(bool)

    # -- multi-round admission (SURVEY 8(f) row 4) -------------------------------------------
    def replay(self, queue=None, after_state=True, priority=False):
        """The reference's pod-at-a-time cycle over the uploaded tables, on the device, in queue order.
        Returns a dict: prefilter / node / ready per queue position and, with after_state, the mutated
        node and group columns (the uploaded tables themselves are left untouched).
        priority=True places each passing pod on its best node under the resource priorities on the live
        state (bs_replay_priority; needs upload_nonzero, weights from set_score_weights) instead of the first
        fitting one; with after_state the dict also holds the live non-zero column node_nonzero [2, N].
        Both walks apply the filters that are on: PodFitsHostPorts on live used ports, and MatchInterPodAffinity on
        live presence that each assumed pod's placed class (upload_interpod_placed) joins."""
        q = None if queue is None else np.ascontiguousarray(queue, dtype=np.uint32)
        n = self.P if q is None else len(q)
        L, N, G = self.n_lanes, self.N, self.G
        out = dict(prefilter=np.zeros(n, np.uint8), node=np.zeros(n, np.int32), ready=np.zeros(n, np.uint8))
        r = capi.ReplayResultC()
        if after_state:
            out.update(node_requested=np.zeros((L, N), np.int64), node_pod_count=np.zeros(N, np.int32),
                       node_req_present=np.zeros(N, np.uint32), group_matched=np.zeros(G, np.uint32),
                       group_flags=np.zeros(G, np.uint8), group_min_res=np.zeros((L, G), np.int64),
                       group_min_res_present=np.zeros(G, np.uint32), group_rep_sel=np.zeros(G, np.uint64),
                       group_rep_tol=np.zeros(G, np.uint64))
        for k, v in out.items():
            setattr(r, k, capi.ptr(v))
        qp = None if q is None else capi.ptr(q)
        if priority:
            nz = np.zeros((2, N), np.int64) if after_state else None
            self._check(self.lib.bs_replay_priority(self.h, qp, n, C.byref(r), None if nz is None else capi.ptr(nz)))
            if after_state:
                out["node_nonzero"] = nz
        else:
            self._check(self.lib.bs_replay(self.h, qp, n, C.byref(r)))
        return out

    # -- preemption ---------------------------------------------------------------------------
    def upload_bound_pods(self, bt: BoundPodTable):
        """The pods bound to the uploaded nodes (upload nodes and groups first; either upload drops this table)."""
        self._check(self.lib.bs_upload_bound_pods(self.h, C.byref(_table_c(bt))))
        self._bound_rows = bt.n

    def upload_bound_host_ports(self, ports):
        """[V] uint64, bit k = bound row v holds entry k of upload_host_ports' dictionary: what preemption under the
        PodFitsHostPorts filter frees when it evicts the row (upload the bound pods first; uploading them again drops
        it).  The bits are checked against the node side when a preemption starts."""
        ports = np.ascontiguousarray(ports, dtype=np.uint64).reshape(-1)
        self._check(self.lib.bs_upload_bound_host_ports(self.h, len(ports), capi.ptr(ports)))

    def _preempt_call(self, pods, victims_cap, call):
        """bs_preempt or bs_preempt_walk as call(pods pointer, n, result) into fresh result arrays, with a first call
        to size the victim list when victims_cap is None: (node, n_victims, n_candidates, victim_offset, victims)."""
        idx = np.ascontiguousarray(pods, dtype=np.uint32)
        n = len(idx)
        node, nv, cand = np.zeros(n, np.int32), np.zeros(n, np.uint32), np.zeros(n, np.uint32)
        off = np.zeros(n + 1, np.uint32)
        cap = 0 if victims_cap is None else victims_cap
        while True:
            vict = np.zeros(max(cap, 1), np.uint32)
            r = capi.PreemptResultC(capi.ptr(node), capi.ptr(nv), capi.ptr(cand), capi.ptr(off), capi.ptr(vict), cap, 0)
            rc = call(capi.ptr(idx) if n else None, n, C.byref(r))
            if rc == capi.BS_E_INVAL and victims_cap is None and r.victims_total > cap:
                cap = r.victims_total
                continue
            self._check(rc)
            return node, nv, cand, off, vict[:r.victims_total].copy()

    def preempt(self, pods, victims_cap=None) -> PreemptResult:
        """For every pod index in `pods`: the node preemption would pick and the pods it would evict there.
        victims_cap: capacity of the victim list (None: as large as the answer needs, found with a first call)."""
        return PreemptResult(*self._preempt_call(pods, victims_cap,
                                                 lambda p, n, r: self.lib.bs_preempt(self.h, p, n, r)))

    def preempt_walk(self, pods, gang=False, victims_cap=None) -> PreemptWalkResult:
        """The preemptors of `pods` one after another in list order (priorities non-increasing), each seeing the
        evictions and nominations of those before it; with `gang`, the preemptors of one group (contiguous in the
        list) are preempted for all together or not at all.  victims_cap as in preempt()."""
        idx = np.ascontiguousarray(pods, dtype=np.uint32)
        outcome, evicted_by = np.zeros(len(idx), np.uint32), np.zeros(self._bound_rows, np.int32)
        flags = capi.PREEMPT_GANG if gang else 0
        res = self._preempt_call(idx, victims_cap, lambda p, n, r: self.lib.bs_preempt_walk(
            self.h, p, n, flags, r, capi.ptr(outcome) if n else None, capi.ptr(evicted_by)))
        return PreemptWalkResult(*res, outcome, evicted_by)

    def remove_pod(self, pod: int, bound: int):
        """batchSchedulingPluginExtension.RemovePod for pod `pod` and bound pod `bound`: (code, reason, group)."""
        st = capi.StatusC()
        self._check(self.lib.bs_remove_pod(self.h, pod, bound, C.byref(st)))
        return st.code, st.reason, st.group

    # -- per-call mirrors ------------------------------------------------------------------
    def prefilter(self, pod: int):
        st = capi.StatusC()
        self._check(self.lib.bs_prefilter(self.h, pod, C.byref(st)))
        return st.code, st.reason, st.group

    def permit(self, pod: int, node: int):
        r = capi.PermitResultC()
        self._check(self.lib.bs_permit(self.h, pod, node, C.byref(r)))
        return dict(ready=bool(r.ready), code=r.code, wait_ns=r.wait_ns, start_signal=bool(r.start_signal),
                    group=r.group)

    # -- gang state: the reference's TTL tables around Permit, kept in the engine --------------------
    def state_reset(self):
        self._check(self.lib.bs_state_reset(self.h))

    def set_pod_ids(self, uid, name_id):
        uid = np.ascontiguousarray(uid, dtype=np.uint64)
        name_id = np.ascontiguousarray(name_id, dtype=np.uint64)
        assert len(uid) == self.P and len(name_id) == self.P
        self._check(self.lib.bs_set_pod_ids(self.h, capi.ptr(uid), capi.ptr(name_id)))

    def begin_cycle(self, now_ns: int):
        self._check(self.lib.bs_begin_cycle(self.h, int(now_ns)))

    def permit_at(self, pod: int, node: int, now_ns: int):
        r = capi.PermitResultC()
        self._check(self.lib.bs_permit_at(self.h, pod, node, int(now_ns), C.byref(r)))
        return dict(ready=bool(r.ready), code=r.code, wait_ns=r.wait_ns, start_signal=bool(r.start_signal), group=r.group)

    def expire(self, now_ns: int, cap: int = None):
        cap = cap or max(self.P, 1)
        rg, ru = np.zeros(cap, np.uint32), np.zeros(cap, np.uint64)
        ev = np.zeros(max(self.G, 1), np.uint32)
        nr, ne = C.c_uint32(), C.c_uint32()
        self._check(self.lib.bs_expire(self.h, int(now_ns), capi.ptr(rg), capi.ptr(ru), cap, C.byref(nr), capi.ptr(ev), len(ev),
                                       C.byref(ne)))
        return list(zip(rg[:nr.value].tolist(), ru[:nr.value].tolist())), ev[:ne.value].tolist()

    def allow_list(self, group: int, now_ns: int, cap: int = None):
        cap = cap or max(self.P, 1)
        u, nd = np.zeros(cap, np.uint64), np.zeros(cap, np.uint32)
        n = C.c_uint32()
        self._check(self.lib.bs_allow_list(self.h, group, int(now_ns), capi.ptr(u), capi.ptr(nd), cap, C.byref(n)))
        return u[:n.value].tolist(), nd[:n.value].tolist()

    def deny(self, group: int, now_ns: int):
        self._check(self.lib.bs_deny(self.h, group, int(now_ns)))

    def mark_permitted(self, uid: int, now_ns: int):
        self._check(self.lib.bs_mark_permitted(self.h, int(uid), int(now_ns)))

    def group_state(self, group: int, now_ns: int):
        m, s, d = C.c_uint32(), C.c_int32(), C.c_int32()
        self._check(self.lib.bs_group_state(self.h, group, int(now_ns), C.byref(m), C.byref(s), C.byref(d)))
        return dict(matched=int(m.value), scheduled=bool(s.value), denied=bool(d.value))

    def less(self, a: int, b: int) -> bool:
        rc = self.lib.bs_less(self.h, a, b)
        if rc < 0:
            self._check(rc)
        return bool(rc)

    def message(self, reason: int, ns_name: str = "", occupied_by: str = "") -> str:
        st = capi.StatusC(0, reason, -1)
        buf = C.create_string_buffer(512)
        self._check(self.lib.bs_format_message(C.byref(st), ns_name.encode(), occupied_by.encode(), buf, 512))
        return buf.value.decode()

    # -- multi-GPU: admit-bitmap all-gather over peer memory ------------------------------------
    def peer_setup(self, rank: int, world: int, words_per_rank: int, all_gather_bytes):
        """Maps every rank's gather buffer into this process.  `all_gather_bytes(b) -> [bytes]*world`
        exchanges the 64-byte IPC handles (e.g. torch.distributed.all_gather_object)."""
        self._check(self.lib.bs_peer_init(self.h, rank, world, words_per_rank))
        buf = (C.c_ubyte * 64)()
        self._check(self.lib.bs_peer_handle(self.h, buf))
        handles = all_gather_bytes(bytes(buf))
        blob = (C.c_ubyte * (64 * world)).from_buffer_copy(b"".join(handles))
        self._check(self.lib.bs_peer_attach(self.h, blob))
        self.peer_world, self.peer_wpr = world, words_per_rank

    def peer_detach(self):
        self._check(self.lib.bs_peer_detach(self.h))

    def peer_join(self):
        """Orders work enqueued on the engine stream after this call behind the last round's gathered words."""
        self._check(self.lib.bs_peer_join(self.h))

    def gathered_admit(self) -> np.ndarray:
        """[world, words_per_rank] uint32: every rank's admit bitmap after the last evaluation."""
        out = np.zeros((self.peer_world, self.peer_wpr), np.uint32)
        self._check(self.lib.bs_fetch_gathered_admit(self.h, capi.ptr(out)))
        return out

    # -- device access / measurement ---------------------------------------------------------
    def device_buffer(self, which: int):
        p, n = C.c_void_p(), C.c_size_t()
        self._check(self.lib.bs_device_buffer(self.h, which, C.byref(p), C.byref(n)))
        return p.value, n.value

    def stream(self) -> int:
        return self.lib.bs_stream(self.h)

    def set_profiling(self, on: bool):
        self._check(self.lib.bs_set_profiling(self.h, int(on)))

    def kernel_ms(self):
        out = {}
        for k, name in enumerate(capi.KERNEL_NAMES):
            ms, n = C.c_float(), C.c_uint32()
            self._check(self.lib.bs_kernel_ms(self.h, k, C.byref(ms), C.byref(n)))
            out[name] = (float(ms.value), int(n.value))
        return out

    def fit_shape(self) -> dict:
        """Lane classes of the last evaluation's fit kernel: LW int64, LN int32, LS int32 in 2^k units."""
        w, n, sc = C.c_uint32(), C.c_uint32(), C.c_uint32()
        self._check(self.lib.bs_fit_shape(self.h, C.byref(w), C.byref(n), C.byref(sc)))
        return {"LW": int(w.value), "LN": int(n.value), "LS": int(sc.value)}

    def fit_lanes(self):
        """(kind [L] uint8, unit [L] uint8) of the last evaluation's fit kernel: kind 0 wide, 1 narrow, 2 scaled;
        unit k of a scaled lane (its values in units of 2^k), 0 otherwise."""
        kind, unit = np.zeros(self.n_lanes, np.uint8), np.zeros(self.n_lanes, np.uint8)
        self._check(self.lib.bs_fit_lanes(self.h, capi.ptr(kind), capi.ptr(unit)))
        return kind, unit

    def sort_shape(self) -> dict:
        """What the last evaluation's queue sort launched: kernel (0 none, 1 single-CTA, 2 persistent lean,
        3 persistent wide), its grid in CTAs, and the radix passes kept for the group and the pod table."""
        k, g, gp, pp = C.c_uint32(), C.c_uint32(), C.c_uint32(), C.c_uint32()
        self._check(self.lib.bs_sort_shape(self.h, C.byref(k), C.byref(g), C.byref(gp), C.byref(pp)))
        return {"kernel": int(k.value), "grid": int(g.value), "group_passes": int(gp.value),
                "pod_passes": int(pp.value)}

    def score_memory(self) -> dict:
        """The memory behind the last evaluation's score matrix (bs_score_memory): supported (the device's
        generic-compression attribute) and compressed (compressible memory, else cudaMalloc)."""
        sup, comp = C.c_uint32(), C.c_uint32()
        self._check(self.lib.bs_score_memory(self.h, C.byref(sup), C.byref(comp)))
        return {"supported": int(sup.value), "compressed": bool(comp.value)}

    def replay_shape(self) -> dict:
        """The regime of the last replay walk (bs_replay_shape): cached (block-summary cache on), fitmask (checkFit
        bits per class), n_rep classes, n_blocks of 1024 nodes, findMaxPG's bucket_size and n_buckets, the final lo
        of the dead-node skip and monotone (no negative fixed-lane request)."""
        names = ("cached", "fitmask", "n_rep", "n_blocks", "bucket_size", "n_buckets", "lo", "monotone")
        v = [C.c_uint32() for _ in names]
        self._check(self.lib.bs_replay_shape(self.h, *[C.byref(x) for x in v]))
        return {k: int(x.value) for k, x in zip(names, v)}

    def score_pitch(self) -> int:
        return int(self.lib.bs_score_pitch(self.h))

    def launch_count(self) -> int:
        return int(self.lib.bs_launch_count(self.h))


def format_remove_message(reason: int, pod_name: str = "", victim_name: str = "", victim_ns_name: str = "",
                          buf_len: int = 512) -> str:
    """The reference's RemovePod error text for a bs_remove_code ("" for REMOVE_ALLOW); needs no engine and no device."""
    lib = capi.load()
    st = capi.StatusC(0, reason, -1)
    buf = C.create_string_buffer(buf_len)
    rc = lib.bs_format_remove_message(C.byref(st), pod_name.encode(), victim_name.encode(), victim_ns_name.encode(),
                                      buf, buf_len)
    if rc != 0:
        raise capi.BsError(rc, lib.bs_strerror(rc).decode())
    return buf.value.decode()


def format_fit_error(counts, n_lanes: int, n_nodes: int, scalar_names=None, buf_len: int = 4096, interpod=None,
                     host_ports=None) -> str:
    """kube-scheduler's FailedScheduling text for one reason row; needs no engine and no device.  scalar_names: the
    names of lanes 4.. (None: "lane<d>").  interpod: the row's companion (E, A, N) from fetch_interpod_reason_rows, whose
    MatchInterPodAffinity entries join the message (bs_format_fit_error_interpod).  host_ports: the row's count from
    fetch_host_port_reason_rows, whose PodFitsHostPorts entry joins it (bs_format_fit_error_filters)."""
    lib = capi.load()
    row = np.ascontiguousarray(counts, dtype=np.uint32)
    if row.shape != (4 + n_lanes,):
        raise ValueError("a reason row has 4 + n_lanes bins")
    names = None
    if scalar_names is not None:
        names = (C.c_char_p * max(1, n_lanes - 4))(*[s.encode() for s in scalar_names])
    buf = C.create_string_buffer(buf_len)
    if host_ports is not None:
        ip = None if interpod is None else np.ascontiguousarray(interpod, dtype=np.uint32)
        if ip is not None and ip.shape != (3,):
            raise ValueError("an inter-pod companion row has 3 counters")
        hp = np.ascontiguousarray(host_ports, dtype=np.uint32).reshape(-1)
        if hp.shape != (1,):
            raise ValueError("a host-port companion row has 1 counter")
        rc = lib.bs_format_fit_error_filters(capi.ptr(row), n_lanes, capi.ptr(ip), capi.ptr(hp), n_nodes,
                                             C.cast(names, C.c_void_p) if names is not None else None, buf, buf_len)
    elif interpod is not None:
        ip = np.ascontiguousarray(interpod, dtype=np.uint32)
        if ip.shape != (3,):
            raise ValueError("an inter-pod companion row has 3 counters")
        rc = lib.bs_format_fit_error_interpod(capi.ptr(row), n_lanes, capi.ptr(ip), n_nodes,
                                              C.cast(names, C.c_void_p) if names is not None else None, buf, buf_len)
    else:
        rc = lib.bs_format_fit_error(capi.ptr(row), n_lanes, n_nodes,
                                     C.cast(names, C.c_void_p) if names is not None else None, buf, buf_len)
    if rc != 0:
        raise capi.BsError(rc, lib.bs_strerror(rc).decode())
    return buf.value.decode()
