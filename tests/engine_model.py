"""TEST INFRASTRUCTURE — a host model of one long-lived engine's logical state, and a seeded generator of call sequences.

Model.apply(op) follows one call: it updates the tables, side columns, filter halves and weights the engine keeps
between calls and returns the error code the engine must answer (None for success).  The drop rules and check orders are
include/bsched.h's; Model.expect(cfg) gives every output of a round on the current state from the existing CPU
restatements only (the oracle, the reason rows, the priority lists, the lane classifier, the walks and preemption).

generate(seed) is a list of ops: random uploads, row updates, side columns, weights, failing calls and rounds, the
MatchInterPodAffinity filter's switch, halves and placed side (all built with one seed, so that they describe one
cluster), the PodFitsHostPorts filter's switch and halves (failing ones too), walks with either filter or both,
bound-pod tables with PodDisruptionBudget bits, preemption and preemption walks (now and then with a list that breaks
one of bs_preempt_walk's rules), plus the scripted bursts R1-R12 (every seed runs at least one; across seeds all of
them, each first in some seed):
  R1  more than 4096 fit and representative classes, then a table with few (both persistent class indices clear),
      then bs_update_groups with a new representative class, then a round;
  R2  node tables of 0, 1, 511, 512, 513 and more nodes, growing and shrinking, every side uploaded again after each;
  R3  one lane narrow -> scaled -> wide through row updates, a row put back (stays wide), a pod table that changes a
      scaled lane's unit, a fresh node table (narrow again);
  R4  each side dropped by the call that owns it: BS_E_STATE with its weight on, the lists without the term with it
      off, and the term back once the side is uploaded again;
  R5  a failing upload of each table kind, then a round;
  R6  every list output at N = 0 and at P = 0 with every term on;
  R7  the filter's lifecycle: the switch without halves, each half dropped by bs_update_nodes, a node table of another
      size and a pod table refused for its lane count and uploaded again, a failing pod half, the four refusals;
  R8  more than 4096 fit classes under the filter, pod halves in new filter classes until the fit class index is
      compacted, the switch toggled, a group row update and an affinity table in between, then a small pod table;
  R9  preemption with budget bits and walks after a group row update, a node row update and a group upload, and one
      walk per broken list rule;
  R10 the ports filter's lifecycle: the switch without halves, each half dropped by the call that owns it, a node
      table of another size, a pod table refused for its lane count followed by another want half and a round, every
      failing node half, a dictionary the want bits pass, preemption refused, the switch off;
  R11 more than 4096 fit classes under the ports filter, want halves in new conflict classes until the fit class index
      is compacted, the inter-pod switch toggled and a group row update in between, then a small pod table;
  R12 walks under the inter-pod filter, the ports filter and both: right after a filter half and before any round,
      after a node row update and the node halves again; the placed side dropped by a refused pod upload, a placed
      term past the filter's dictionary, and the placed side not read with the filter off.
"""
from __future__ import annotations

import numpy as np

import fit_reasons_ref as frr
import fit_shape_cases as fsc
import host_ports_ref as hr
import interpod_filter_ref as fr
import interpod_priority_ref as ir
import interpod_walk_ref as iwr
import locality_priority_ref as lpr
import preempt_pdb_ref
import preempt_walk_ref as pwr
import ratio_priority_ref as rr
from oracle import oracle
from randsnap import S, random_snapshot

E_INVAL, E_RANGE, E_STATE, E_INDEX = -1, -5, -6, -8
I64_MIN = np.iinfo(np.int64).min
LIMIT = 1 << 56
NODE_SIDES = ("nz_node", "pref_node", "loc_node", "spread_node", "ipa_node")
POD_SIDES = ("nz_pod", "pref_pod", "loc_pod", "spread_pod", "ipa_pod")
PW, LW, W_SPREAD, W_IPA = (1, 1), (1, 10000), 1, 1
RATIO_ON = (2, rr.BIN_PACK, None, 1)   # lane weights filled in per lane count
AFF = 3   # affinity classes of every generated table: pods and groups name classes 0..2 of each node upload's table


def expected_topk(score, K):
    """[P, N] oracle scores (INT64_MIN = does not fit) -> (nodes [P, K] int32, scores [P, K] int64): each row's fitting
    entries by score descending, then node index ascending, cut to K, padded with node -1 and score INT64_MIN."""
    P, N = score.shape
    nodes = np.full((P, K), -1, np.int32)
    scores = np.full((P, K), I64_MIN, np.int64)
    if N == 0:
        return nodes, scores
    fit = score != I64_MIN
    key = np.where(fit, score, -1)                     # fitting scores are >= 0
    idx = np.broadcast_to(np.arange(N), (P, N))
    order = np.lexsort((idx, -key), axis=1)[:, :K]
    take = min(K, N)
    ok = np.take_along_axis(fit, order, axis=1)
    nodes[:, :take] = np.where(ok, order, -1)
    scores[:, :take] = np.where(ok, np.take_along_axis(score, order, axis=1), I64_MIN)
    return nodes, scores


def _out_of_range(*arrays):
    return any(np.size(a) and (np.abs(np.asarray(a, np.int64)) > LIMIT).any() for a in arrays)


def _apply_rows(table, idx, rows):
    """A copy of `table` with rows idx overwritten by the compact table `rows` (the same layout)."""
    out = table.copy()
    for f in out.__dataclass_fields__:
        a, r = getattr(out, f), getattr(rows, f)
        if a is None or r is None:
            continue
        if a.ndim == 2:
            a[:, idx] = r
        else:
            a[idx] = r
    return out


def _or(masks):
    """The OR of a uint64 mask column, as a Python int."""
    return int(np.bitwise_or.reduce(np.asarray(masks, np.uint64).reshape(-1), initial=np.uint64(0)))


def no_interpod_filter(N, P):
    """((node, pods), placed): MatchInterPodAffinity filter columns without a term, every pod without a class and a
    placed side without a class.  interpod_walk_ref.replay passes every node with them, so that it walks the ports
    filter alone around any chooser."""
    none = np.full(P, S.IPF_NONE, np.uint32)
    u32 = lambda n: np.zeros(n, np.uint32)
    node = (u32(0), np.zeros((0, N), np.uint32), u32(0), u32(0), u32(0),
            (u32(1), u32(0), np.zeros(0, np.int32), np.zeros(0, np.uint8)))
    pods = (none, (u32(1), u32(0), np.zeros(0, np.uint8), np.zeros(0, np.uint8)))
    return (node, pods), (none.copy(), (u32(1), u32(0), np.zeros(0, np.int32), np.zeros(0, np.uint8)))


def _max_class(cls, none):
    c = np.asarray(cls, np.int64)
    c = c[c != none]
    return int(c.max()) if c.size else -1


class Model:
    """The logical state of one engine with `lanes` lanes (see the module docstring)."""

    def __init__(self, lanes):
        self.lanes = lanes
        self.nodes = self.pods = self.groups = None
        self.aff = None          # [n_aff, W] bits, or None (no table: n_aff = 0)
        self.bound = None
        self.history = []        # node tables replaced by row updates since the last full node upload
        self.side = dict.fromkeys(NODE_SIDES + POD_SIDES)
        self.weights = (1, 0, 1)
        self.ratio = ir.NO_RATIO
        self.pw, self.lw, self.w_spread, self.w_ipa = (0, 0), (0, 0), 0, 0
        # the MatchInterPodAffinity filter: the switch, its two halves (node: the node side's columns, pod: (pod_class,
        # class table)), and whether the last successful round ran with the switch on (else its companion rows are 0)
        self.ipf_on, self.ipf_node, self.ipf_pod, self.ipf_round = False, None, None, False
        # the filter's placed side (pod_class, class table): what the walks add to presence for each pod they assume
        self.ipf_placed = None
        # the PodFitsHostPorts filter: the switch, its two halves (node: (entries [K, 3], used [N]), pod: want [P]) and
        # whether the last successful round ran with it on (else its companion rows are 0)
        self.hp_on, self.hp_node, self.hp_pod, self.hp_round = False, None, None, False

    # ---- state ---------------------------------------------------------------------------------------------------
    def snapshot(self):
        return S.Snapshot(self.nodes, self.pods, self.groups, aff_bits=self.aff)

    def complete(self):
        return self.nodes is not None and self.pods is not None and self.groups is not None

    def _drop(self, keys):
        for k in keys:
            self.side[k] = None

    # ---- one call ------------------------------------------------------------------------------------------------
    def apply(self, op):
        kind = op["op"]
        f = getattr(self, "_" + kind, None)
        if f is None:
            raise ValueError(kind)
        return f(op)

    def _upload_nodes(self, op):
        nt = op["table"]
        self._drop(NODE_SIDES)
        self.ipf_node = self.hp_node = None
        self.bound, self.aff = None, None   # they belong to the snapshot, also to one that fails validation
        if _out_of_range(nt.alloc, nt.requested):
            self.nodes = None
            return E_RANGE
        self.nodes, self.history = nt, []
        return None

    def _update_nodes(self, op):
        idx, rows = op["idx"], op["rows"]
        if self.nodes is None:
            return E_STATE
        self._drop(NODE_SIDES)   # every call, also one that changes no row or fails (bsched.h bs_update_nodes)
        self.ipf_node = self.hp_node = None
        if len(idx) == 0:
            return None
        if (np.asarray(idx) >= self.nodes.n).any():
            return E_INDEX
        if _out_of_range(rows.alloc, rows.requested):
            return E_RANGE
        self.history.append(self.nodes)
        self.nodes = _apply_rows(self.nodes, idx, rows)
        self.bound = None
        return None

    def _upload_groups(self, op):
        gt = op["table"]
        self.bound = None
        if _out_of_range(gt.min_res):
            self.groups = None
            return E_RANGE
        self.groups = gt
        return None

    def _update_groups(self, op):
        idx, rows = op["idx"], op["rows"]
        if self.groups is None:
            return E_STATE
        if len(idx) == 0:
            return None
        if (np.asarray(idx) >= self.groups.n).any():
            return E_INDEX
        if _out_of_range(rows.min_res):
            return E_RANGE
        self.groups = _apply_rows(self.groups, idx, rows)   # the bound-pod table stays
        return None

    def _upload_pods(self, op):
        pt = op["table"]
        self._drop(POD_SIDES)
        self.ipf_pod = self.ipf_placed = self.hp_pod = None   # also by a call refused for its lane count, which keeps
        # the pod table of now
        if pt.lanes != self.lanes:
            return E_INVAL
        if _out_of_range(pt.req):
            self.pods = None
            return E_RANGE
        self.pods = pt
        return None

    def _upload_affinity(self, op):
        if self.nodes is None:
            return E_STATE
        bits = op["bits"]
        self.aff = None if bits is None or len(bits) == 0 else bits
        return None

    def _upload_bound(self, op):
        if self.nodes is None:
            return E_STATE
        self.bound = op["table"]
        return None

    def _side(self, op):
        """One half of a side: name (nz / pref / loc / spread / ipa), half (node / pod), cols, n (its length)."""
        key = op["name"] + "_" + op["half"]
        self.side[key] = None    # a failing call leaves the side dropped
        table = self.nodes if op["half"] == "node" else self.pods
        if table is None:
            return E_STATE
        if op["n"] != table.n:
            return E_INVAL
        self.side[key] = op["cols"]
        return None

    def _ipf(self, op):
        """One half of the filter's columns: half (node / pod), cols, n (its length)."""
        key = "ipf_" + op["half"]
        setattr(self, key, None)   # a failing call leaves the half dropped
        table = self.nodes if op["half"] == "node" else self.pods
        if table is None:
            return E_STATE
        if op["n"] != table.n:
            return E_INVAL
        if op["half"] == "pod" and _max_class(op["cols"][0], S.IPF_NONE) >= len(op["cols"][1][0]) - 1:
            return E_INDEX
        if op["half"] == "node" and (np.asarray(op["cols"][3], np.int64) >= table.n).any():
            return E_INDEX     # a bound pod on a node the table lacks
        setattr(self, key, op["cols"])
        return None

    def _ipf_switch(self, op):
        self.ipf_on = bool(op["on"])
        return None

    def _placed(self, op):
        """The filter's placed side: cols = (pod_class, (class_offset, term, own, match)), n (its length)."""
        self.ipf_placed = None   # a failing call leaves it dropped
        if self.pods is None:
            return E_STATE
        if op["n"] != self.pods.n:
            return E_INVAL
        pcls, (off, _, own, _) = op["cols"]
        if _max_class(pcls, S.IPF_NONE) >= len(off) - 1:
            return E_INDEX
        if not np.isin(np.asarray(own, np.int64), (0, 1)).all():
            return E_RANGE
        self.ipf_placed = op["cols"]
        return None

    def _hp(self, op):
        """One half of the ports filter's columns: half (node: cols = (entries [K, 3], used [N]); pod: cols = want
        [P]), n (its length).  The node half's checks in the engine's order: the length, more than 64 entries, a port
        outside 1..65535, an entry listed twice, a used bit past the entries."""
        key = "hp_" + op["half"]
        setattr(self, key, None)   # a failing call leaves the half dropped
        table = self.nodes if op["half"] == "node" else self.pods
        if table is None:
            return E_STATE
        if op["n"] != table.n:
            return E_INVAL
        if op["half"] == "node":
            ent = np.asarray(op["cols"][0], np.int64).reshape(-1, 3)
            K = len(ent)
            if K > 64:
                return E_INVAL
            if ((ent[:, 2] < 1) | (ent[:, 2] > 65535)).any():
                return E_RANGE
            if len(set(map(tuple, ent.tolist()))) < K:
                return E_INVAL
            if K < 64 and _or(op["cols"][1]) >> K:
                return E_INDEX
        setattr(self, key, op["cols"])
        return None

    def _hp_switch(self, op):
        self.hp_on = bool(op["on"])
        return None

    def _weights(self, op):
        for k, v in op.items():
            if k != "op":
                setattr(self, k, v)
        return None

    def _evaluate(self, op):
        rc = self._evaluate_check(op)
        if rc is None:
            self.ipf_round, self.hp_round = self.ipf_on, self.hp_on
        return rc

    def _evaluate_check(self, op):
        """The engine's check order: the tables, then (priority lists only) the non-zero columns, the node
        priorities, locality, spread and inter-pod, then the filter's halves and terms, then the affinity class ids."""
        if not self.complete():
            return E_STATE
        if op["priority"]:
            sd = self.side
            if sd["nz_node"] is None or sd["nz_pod"] is None:
                return E_STATE
            if any(self.pw):
                if sd["pref_node"] is None or sd["pref_pod"] is None:
                    return E_STATE
                if self.pw[1] and _max_class(sd["pref_pod"][1], S.PREF_NONE) >= sd["pref_node"][1].shape[0]:
                    return E_INDEX
            rc = self._locality_check()
            if rc:
                return rc
            if self.w_spread:
                if sd["spread_node"] is None or sd["spread_pod"] is None:
                    return E_STATE
                if _max_class(sd["spread_pod"], S.SPREAD_NONE) >= sd["spread_node"][1].shape[0]:
                    return E_INDEX
            if self.w_ipa:
                if sd["ipa_node"] is None or sd["ipa_pod"] is None:
                    return E_STATE
                if _max_class(sd["ipa_pod"][1][1], -1) >= len(sd["ipa_node"][2]):
                    return E_INDEX
        rc = (self.ipf_on and self._interpod_filter_check()) or (self.hp_on and self._host_port_check())
        return rc or self._affinity_check()

    def _interpod_filter_check(self):
        if self.ipf_node is None or self.ipf_pod is None:
            return E_STATE
        if _max_class(self.ipf_pod[1][1], -1) >= len(self.ipf_node[2]):   # any class's term, used or not
            return E_INDEX
        return None

    def _host_port_check(self):
        if self.hp_node is None or self.hp_pod is None:
            return E_STATE
        K = len(np.asarray(self.hp_node[0]).reshape(-1, 3))
        if K < 64 and _or(self.hp_pod) >> K:   # a want bit past the node half's entries
            return E_INDEX
        return None

    def _locality_check(self):
        sd = self.side
        if self.lw[0]:
            if sd["loc_node"] is None or sd["loc_pod"] is None:
                return E_STATE
            cls, off, ids, _ = sd["loc_pod"]
            if _max_class(cls, S.IMAGE_NONE) >= len(off) - 1 or _max_class(ids, -1) >= len(sd["loc_node"][0]):
                return E_INDEX
        if self.lw[1] and (sd["loc_node"] is None or sd["loc_pod"] is None):
            return E_STATE
        return None

    def _affinity_check(self):
        n_aff = 0 if self.aff is None else len(self.aff)
        for a in (self.pods.aff_class, self.groups.rep_aff):
            if a is not None and _max_class(a, S.AFF_NONE) >= n_aff:
                return E_INDEX
        return None

    def _replay(self, op):
        """bs_replay / bs_replay_priority (engine.cu replay_walk): the filter on without the placed side and then
        bs_replay_priority's weights before anything else; the tables, the non-zero columns, locality, the ports
        filter, the inter-pod filter, a placed term past the filter's dictionary, then the affinity class ids."""
        if self.ipf_on and self.ipf_placed is None:
            return E_INVAL
        if op["priority"] and (any(self.pw) or self.w_spread or self.w_ipa):
            return E_INVAL
        if not self.complete():
            return E_STATE
        if op["priority"]:
            if self.side["nz_node"] is None or self.side["nz_pod"] is None:
                return E_STATE
            rc = self._locality_check() if any(self.lw) else None
            if rc:
                return rc
        rc = (self.hp_on and self._host_port_check()) or (self.ipf_on and self._interpod_filter_check())
        if rc:
            return rc
        if self.ipf_on and _max_class(self.ipf_placed[1][1], -1) >= len(self.ipf_node[2]):
            return E_INDEX
        return self._affinity_check()

    def _preempt(self, op):
        """bs_preempt's checks (preempt_prologue in engine.cu): the filters' switches, the tables, then each listed
        pod's index and affinity class."""
        if self.ipf_on or self.hp_on:
            return E_INVAL
        if not self.complete() or self.bound is None:
            return E_STATE
        pods = np.asarray(op["pods"], np.int64)
        if (pods >= self.pods.n).any():
            return E_INDEX
        n_aff = 0 if self.aff is None else len(self.aff)
        if self.pods.aff_class is not None and _max_class(self.pods.aff_class[pods], S.AFF_NONE) >= n_aff:
            return E_INDEX
        return None

    def _preempt_walk(self, op):
        """bs_preempt's checks, then the list rules in the engine's order (include/bsched.h bs_preempt_walk): per list
        position, a priority above the one before, a pod listed twice, and with gang a group (0 <= gid < n_groups)
        whose run started before and was closed."""
        rc = self._preempt(op)
        if rc:
            return rc
        pods = np.asarray(op["pods"], np.int64)
        prio, gid, G = self.pods.priority[pods], self.pods.gid[pods], self.groups.n
        seen, closed = set(), set()
        for i, p in enumerate(pods.tolist()):
            if i and prio[i] > prio[i - 1]:
                return E_INVAL
            if p in seen:
                return E_INVAL
            seen.add(p)
            if not op["gang"] or not 0 <= gid[i] < G or (i and gid[i - 1] == gid[i]):
                continue
            if gid[i] in closed:
                return E_INVAL
            closed.add(gid[i])
        # the generator stays under the walk's BS_E_RANGE bound: every value is within +-LIMIT, so the live sums are
        # at most (4 + n) * LIMIT plus the pod counts
        pc = max([int(t.pod_count.max()) for t in self.history + [self.nodes] if t.n] + [0])
        assert (4 + len(pods)) * LIMIT + pc + len(pods) <= 1 << 62, "a walk the engine refuses with BS_E_RANGE"
        return None

    # ---- what a round gives ----------------------------------------------------------------------------------------
    def priority_rows(self, K, pods=None, snap=None):
        sd, snap = self.side, snap or self.snapshot()
        N, P = self.nodes.n, self.pods.n
        zero = (([1], [np.zeros(N)], [0], [], [], ([0], [], [], [])), (np.full(P, S.IPA_NONE), ([0], [], [], [])))
        interpod = (sd["ipa_node"], sd["ipa_pod"]) if self.w_ipa else zero
        prefs = sd["pref_node"] + sd["pref_pod"] if any(self.pw) else None
        loc = (sd["loc_node"], sd["loc_pod"]) if any(self.lw) else None
        spread = (sd["spread_node"], sd["spread_pod"]) if self.w_spread else None
        ratio = self.ratio_setting()
        return ir.priority_rows(snap, sd["nz_node"], sd["nz_pod"], K, interpod, self.w_ipa, ratio, self.weights, prefs,
                                self.pw, loc, self.lw, spread, self.w_spread, pods=pods)

    def ratio_setting(self):
        return self.ratio if self.ratio[0] else ir.NO_RATIO

    def expect(self, cfg):
        """Every output of a round on this state for an engine built with cfg (score, fit_bitmap, filter, reasons,
        topk, priority_k): a dict of arrays, keyed as the GPU test reads them back.  With the filter on, the round is
        interpod_filter_ref.expected_round's, with the ports filter on host_ports_ref.expected_round's (with the
        inter-pod verdicts when both are on); interpod_rows and host_port_rows (with reasons) are the companion rows,
        zero when the last round ran with that filter off."""
        snap = self.snapshot()
        if self.ipf_round or self.hp_round:
            def lists(fsnap, score):
                out = {}
                if cfg.get("topk"):
                    out["topk_nodes"], out["topk_scores"] = expected_topk(score, cfg["topk"])
                if cfg.get("priority_k"):
                    out["priority_nodes"], out["priority_scores"] = self.priority_rows(cfg["priority_k"], snap=fsnap)
                return out
            ipf = (self.ipf_node, self.ipf_pod)
            if self.hp_round:
                (entries, used), want = self.hp_node, self.hp_pod
                ipf_v = fr.verdicts(ipf, self.nodes.n) if self.ipf_round else None
                out, _ = hr.expected_round(snap, hr.passes(entries, used, want), cfg, lists, ipf_v)
            else:
                out, _ = fr.expected_round(snap, ipf, cfg, lists)
            if cfg.get("reasons"):
                out.setdefault("interpod_rows", np.zeros((self.pods.n, 3), np.uint32))
                out.setdefault("host_port_rows", np.zeros(self.pods.n, np.uint32))
            out["lanes"] = fsc.classify(self.nodes, self.pods, self.history)
            return out
        orc = oracle.round(snap, want_bitmap=True, want_score=True, want_filter=cfg.get("filter", False))
        out = {f: getattr(orc, f) for f in ("prefilter", "feasible_count", "best_node", "best_score", "admit",
                                             "admit_bitmap", "new_denied", "order", "rank")}
        out["max_group"], out["max_finished"] = orc.max_group, orc.max_finished
        if cfg.get("fit_bitmap"):
            out["fit_rows"] = orc.fit_bitmap
        if cfg.get("score"):
            out["score_rows"] = orc.score
        if cfg.get("filter"):
            out["filter_rows"], out["filter_code"] = orc.filter_bitmap, orc.filter_code
        if cfg.get("topk"):
            out["topk_nodes"], out["topk_scores"] = expected_topk(orc.score, cfg["topk"])
        if cfg.get("reasons"):
            out["reason_rows"] = frr.fit_reasons(snap)
            out["interpod_rows"] = np.zeros((self.pods.n, 3), np.uint32)
            out["host_port_rows"] = np.zeros(self.pods.n, np.uint32)
        if cfg.get("priority_k"):
            out["priority_nodes"], out["priority_scores"] = self.priority_rows(cfg["priority_k"])
        out["lanes"] = fsc.classify(self.nodes, self.pods, self.history)
        return out

    def expect_walk(self, priority, queue):
        """The walk on this state: with either filter on interpod_walk_ref.replay (with the ports filter inside it;
        with the inter-pod filter off, one without terms), else the oracle's walk or bs_replay_priority's."""
        snap = self.snapshot()
        sd = self.side
        loc = None
        if priority:
            loc = (sd["loc_node"], sd["loc_pod"]) if any(self.lw) else \
                ((np.zeros(0, np.int64), np.zeros((0, (self.nodes.n + 31) // 32), np.uint32),
                  np.zeros(self.nodes.n, np.uint64)),
                 (np.full(self.pods.n, S.IMAGE_NONE, np.uint32), np.zeros(1, np.uint32), np.zeros(0, np.uint32),
                  np.full(self.pods.n, S.AVOID_NONE, np.uint8)))
        if self.ipf_on or self.hp_on:
            cols, placed = ((self.ipf_node, self.ipf_pod), self.ipf_placed) if self.ipf_on else \
                no_interpod_filter(self.nodes.n, self.pods.n)
            nz = (sd["nz_node"], sd["nz_pod"]) if priority else None
            hp = (self.hp_node, self.hp_pod) if self.hp_on else None
            pf, node, ready, _, _, _ = iwr.replay(snap, cols, placed, queue, nz, self.weights, self.ratio_setting(), loc,
                                                  self.lw, hp)
        elif priority:
            pf, node, ready, _, _ = lpr.replay_locality(snap, sd["nz_node"], sd["nz_pod"], loc, self.lw,
                                                        self.ratio_setting(), queue, self.weights)
        else:
            pf, node, ready, _ = oracle.replay(snap, queue)
        return {"prefilter": pf, "node": node, "ready": ready}

    def expect_preempt(self, pods):
        r = preempt_pdb_ref.preempt(self.snapshot(), self.bound, pods)
        return {"node": r.node, "n_victims": r.n_victims, "n_candidates": r.n_candidates, "victims": r.victims}

    def expect_preempt_walk(self, pods, gang):
        r = pwr.walk(self.snapshot(), self.bound, pods, gang)
        return {"node": r.node, "n_victims": r.n_victims, "n_candidates": r.n_candidates, "victims": r.victims,
                "outcome": r.outcome, "evicted_by": r.evicted_by}


# ---- the generator -----------------------------------------------------------------------------------------------

def describe(op):
    """One line per op for a failure report."""
    parts = [op["op"]]
    for k, v in op.items():
        if k == "op":
            continue
        if hasattr(v, "n") and hasattr(v, "lanes"):
            parts.append(f"{k}=<{type(v).__name__} n={v.n}>")
        elif isinstance(v, np.ndarray):
            parts.append(f"{k}=<{v.dtype}[{','.join(map(str, v.shape))}]>")
        elif k == "cols":
            parts.append("cols=...")
        else:
            parts.append(f"{k}={v!r}")
    return " ".join(parts)


class Generator:
    """Seeded op sequences over one lane count; the burst methods append scripted regimes."""

    def __init__(self, seed, lanes=6):
        self.seed, self.L = seed, lanes
        self.rng = np.random.default_rng(seed)
        self.model = Model(lanes)   # the generator's own copy: side columns are built on the state of now
        self.ops = []
        self.regimes = set()
        self.max_p = 0
        self.ipf_seed = seed   # both filter halves and the placed side are built with it: they describe one cluster
        self.hp_seed = seed    # both ports halves are built with it: they draw the same dictionary

    def _k(self):
        return int(self.rng.integers(0, 1 << 30))

    def emit(self, op):
        self.model.apply(op)
        self.ops.append(op)
        return op

    # -- tables --
    def snap(self, P, N, G, aff=0, case=None):
        return random_snapshot(self._k(), P=P, N=N, G=G, L=self.L, case=case or str(self.rng.choice(["mixed", "A", "B"])),
                               aff=aff)

    def upload_nodes(self, N, aff=AFF):
        s = self.snap(1, N, 1, aff=aff)
        self.emit({"op": "upload_nodes", "table": s.nodes})
        if aff and s.aff_bits is not None:
            self.emit({"op": "upload_affinity", "bits": s.aff_bits})

    def upload_pods(self, P, aff=AFF):
        m = self.model
        G = m.groups.n if m.groups is not None else 8
        s = self.snap(P, 1, max(G, 1), aff=aff)
        pt = s.pods
        if G == 0:
            pt.gid[:] = np.where(pt.gid >= 0, 3, pt.gid)   # out-of-range gids: the oracle treats them as missing
        self.max_p = max(self.max_p, P)
        self.emit({"op": "upload_pods", "table": pt})

    def upload_groups(self, G, aff=AFF):
        s = self.snap(1, 1, G, aff=aff)
        self.emit({"op": "upload_groups", "table": s.groups})

    def update_nodes(self, mode):
        m = self.model
        N = m.nodes.n
        k = int(self.rng.integers(1, min(N, 9) + 1))
        idx = np.sort(self.rng.choice(N, k, replace=False)).astype(np.uint32)
        rows = m.nodes.take(idx).copy()
        if mode == "widen":
            rows.alloc[0, 0] = 1 << 40
        elif mode == "back":
            rows = self._first.take(idx).copy() if getattr(self, "_first", None) is not None and \
                self._first.n == N else rows
        elif mode == "flags":
            rows.flags[:] = self.rng.choice([0, S.NODE_UNSCHEDULABLE, S.NODE_NIL, S.NODE_TAINTS_ERR], k)
        elif mode == "labels":
            rows.label_mask[:] = self.rng.integers(0, 16, k)
            rows.taint_mask[:] = self.rng.integers(0, 4, k)
        self.emit({"op": "update_nodes", "idx": idx, "rows": rows, "mode": mode})

    def update_groups(self, mode):
        m = self.model
        G = m.groups.n
        k = int(self.rng.integers(1, min(G, 6) + 1))
        idx = np.sort(self.rng.choice(G, k, replace=False)).astype(np.uint32)
        rows = m.groups.take(idx).copy()
        if mode == "rep":
            rows.rep_sel[0] = np.uint64(0xF0F0 + int(self.rng.integers(0, 1 << 12)))
            rows.flags[0] |= S.GROUP_HAS_POD
        else:
            rows.creation_ns[0] = np.int64(1) << int(self.rng.integers(40, 62))
            rows.matched[:] = self.rng.integers(0, 3, k)
        self.emit({"op": "update_groups", "idx": idx, "rows": rows})

    # -- sides --
    def _now(self):
        """The snapshot of now, with empty tables for the missing ones."""
        m = self.model
        return S.Snapshot(m.nodes if m.nodes is not None else S.NodeTable.empty(0, self.L),
                          m.pods if m.pods is not None else S.PodTable.empty(0, self.L),
                          m.groups if m.groups is not None else S.GroupTable.empty(0, self.L))

    def side(self, name, half, mismatch=False, wrong_len=False):
        m = self.model
        table = m.nodes if half == "node" else m.pods
        if table is None:
            return
        snap = self._now()
        k = self._k()
        if name == "nz":
            cols = S.nonzero_requests(snap, k)[0 if half == "node" else 1]
            n = cols.shape[1]
        elif name == "pref":
            c = S.node_preferences(snap, k, n_classes=2 if mismatch else 5)
            cols = (c[0], c[1]) if half == "node" else (c[2], c[3])
            n = len(cols[0])
        elif name == "loc":
            node, pods = S.node_locality(snap, k, n_images=3 if mismatch else 16)
            cols = node if half == "node" else pods
            n = len(node[2]) if half == "node" else len(pods[0])
        elif name == "spread":
            node, pods = S.node_spread(snap, k, n_classes=2 if mismatch else 6)
            cols = node if half == "node" else pods
            n = len(node[0]) if half == "node" else len(pods)
        else:
            node, pods = S.node_interpod(snap, k, n_terms=3 if mismatch else 24)
            cols = node if half == "node" else pods
            n = table.n
        if wrong_len and name in ("nz", "spread"):   # one entry too many
            n += 1
            if name == "nz":
                cols = np.concatenate([cols, np.zeros((2, 1), np.int64)], axis=1)
            elif half == "node":
                cols = (np.r_[cols[0], np.uint8(S.ZONE_NONE)].astype(np.uint8),
                        np.concatenate([cols[1], np.zeros((cols[1].shape[0], 1), np.int32)], axis=1))
            else:
                cols = np.r_[cols, np.uint32(S.SPREAD_NONE)].astype(np.uint32)
        self.emit({"op": "side", "name": name, "half": half, "n": n, "cols": cols, "wrong_len": wrong_len})

    def all_sides(self, halves=("node", "pod")):
        for name in ("nz", "pref", "loc", "spread", "ipa"):
            for half in halves:
                self.side(name, half)
        for half in halves:
            self.ipf(half)
            self.hp(half)
        if "pod" in halves:
            self.placed()

    def node_sides(self):
        """The node halves again (the filter's too), as a caller does after bs_update_nodes dropped them."""
        self.all_sides(("node",))

    def ipf(self, half, mismatch=False, wrong_len=False, bad=False, spread=0):
        """One half of the filter's columns, built from the state of now with the seed of the pod half (another seed
        with mismatch); wrong_len: one entry too many; bad: a pod class out of range; spread > 0: the pod half's class
        table repeated `spread` times and each pod in a random copy of its class (verdicts unchanged, new fit classes)."""
        m = self.model
        table = m.nodes if half == "node" else m.pods
        if table is None:
            return
        node, pods = S.node_interpod_filter(self._now(), self._k() if mismatch else self.ipf_seed)
        if half == "node":
            nv, topo, tkey, bnode, bcls, bcl = node
            if not m.nodes.n:   # the generator puts bound pods on node 0 of an empty table: none can be bound
                bnode, bcls = bnode[:0], bcls[:0]
            rest = (tkey, bnode, bcls, bcl)
            if wrong_len:
                topo = np.concatenate([topo, np.zeros((topo.shape[0], 1), np.uint32)], axis=1)
            cols, n = (nv, topo, *rest), topo.shape[1]
        else:
            pcls, (off, term, role, selfm) = pods
            C = len(off) - 1
            if spread and C:
                pcls = np.where(pcls == S.IPF_NONE, pcls, pcls + C * self.rng.integers(0, spread, len(pcls))).astype(np.uint32)
                off = np.concatenate([off[:1]] + [off[1:] + k * off[-1] for k in range(spread)]).astype(np.uint32)
                term, role, selfm = np.tile(term, spread), np.tile(role, spread), np.tile(selfm, spread)
            if bad:
                pcls = np.full(len(pcls), len(off) - 1, np.uint32)
            if wrong_len:
                pcls = np.r_[pcls, np.uint32(S.IPF_NONE)].astype(np.uint32)
            cols, n = (pcls, (off, term, role, selfm)), len(pcls)
        self.emit({"op": "ipf", "half": half, "n": n, "cols": cols})

    def hp(self, half, wrong_len=False, bad=None, n_entries=12):
        """One half of the ports filter's columns: host_ports_ref.random_columns on the state of now with hp_seed (both
        halves draw the same dictionary first, so a node half of fewer n_entries is a prefix of it); wrong_len: one
        entry too many; bad (node half): "port" (a port 0), "twice" (an entry listed twice), "used" (a used bit past
        the entries) or "many" (65 entries)."""
        m = self.model
        table = m.nodes if half == "node" else m.pods
        if table is None:
            return
        (entries, used), want = hr.random_columns(self._now(), self.hp_seed, n_entries=n_entries)
        if half == "pod":
            cols = np.r_[want, np.uint64(0)].astype(np.uint64) if wrong_len else want
            self.emit({"op": "hp", "half": half, "n": len(cols), "cols": cols})
            return
        entries, used = entries.copy(), used.copy()
        if bad == "port":
            entries[-1, 2] = 0
        elif bad == "twice":
            entries[-1] = entries[0]
        elif bad == "used" and len(used):
            used[-1] |= np.uint64(1) << np.uint64(len(entries))
        elif bad == "many":
            entries = np.array([(1, 0, 1000 + k) for k in range(65)], np.int64)
        if wrong_len:
            used = np.r_[used, np.uint64(0)].astype(np.uint64)
        self.emit({"op": "hp", "half": half, "n": len(used), "cols": (entries, used), "bad": bad})

    def placed(self, wrong_len=False, bad=None):
        """The filter's placed side from snapshot.node_interpod_walk on the state of now with ipf_seed (the draws of
        the filter's halves); wrong_len: one entry too many; bad: "class" (a pod class out of range), "own" (an own of
        2) or "term" (a term one past the node half's dictionary, or past 24 terms without one)."""
        m = self.model
        if m.pods is None:
            return
        pcls, (off, term, own, match) = S.node_interpod_walk(self._now(), self.ipf_seed)[2]
        if bad == "class":
            pcls = np.full(len(pcls), len(off) - 1, np.uint32)
        elif bad in ("own", "term"):   # one more class of one entry, the last pod in it
            T = len(m.ipf_node[2]) if m.ipf_node is not None else 24
            off, term = np.r_[off, off[-1] + 1].astype(np.uint32), np.r_[term, T if bad == "term" else 0].astype(np.uint32)
            own, match = np.r_[own, 2 if bad == "own" else 0].astype(np.int32), np.r_[match, 1].astype(np.uint8)
            if len(pcls):
                pcls = pcls.copy()
                pcls[-1] = len(off) - 2
        if wrong_len:
            pcls = np.r_[pcls, np.uint32(S.IPF_NONE)].astype(np.uint32)
        self.emit({"op": "placed", "n": len(pcls), "cols": (pcls, (off, term, own, match)), "bad": bad})

    def switch(self, on):
        self.emit({"op": "ipf_switch", "on": on})

    def hp_switch(self, on):
        self.emit({"op": "hp_switch", "on": on})

    def walk_weights(self):
        """The weights bs_replay_priority refuses set to 0 (the resource, ratio and locality terms stay)."""
        self.emit({"op": "weights", "pw": (0, 0), "w_spread": 0, "w_ipa": 0})

    def weights(self, on):
        L = self.L
        ratio = (RATIO_ON[0], RATIO_ON[1], [1, 1, 0, 0] + [1] * (L - 4), RATIO_ON[3]) if on else ir.NO_RATIO
        self.emit({"op": "weights", "weights": (1, 0, 1) if on else (2, 1, 3), "ratio": ratio,
                   "pw": PW if on else (0, 0), "lw": LW if on else (0, 0), "w_spread": W_SPREAD if on else 0,
                   "w_ipa": W_IPA if on else 0})

    def round(self, how=None):
        how = how or str(self.rng.choice(["evaluate", "view", "async"]))
        self.emit({"op": "evaluate", "how": how, "priority": True})

    def walk(self, kind):
        if kind == "preempt":
            if self.model.complete():
                self.bound()
            self.emit({"op": "preempt", "pods": np.arange(min(self.model.pods.n if self.model.pods is not None else 0, 40),
                                                         dtype=np.uint32)})
        else:
            self.emit({"op": "replay", "priority": kind == "priority"})

    def bound(self):
        """A bound-pod table of the snapshot of now; none, some or all of its pods violate a PodDisruptionBudget."""
        v = float(self.rng.choice([0.0, 0.3, 1.0]))
        self.emit({"op": "upload_bound", "table": S.bound_pods(self.model.snapshot(), self._k(), max_per_node=6,
                                                               violating=v)})

    def walk_list(self, gang, n=24):
        """Up to n pods in queue order (priority descending, then group, then index); with gang, a group whose members
        the priorities split keeps its first run only, so that the list keeps bs_preempt_walk's rules."""
        pt, G = self.model.pods, self.model.groups.n
        pick = np.sort(self.rng.choice(pt.n, min(n, pt.n), replace=False)) if pt.n else np.zeros(0, np.int64)
        pick = pick[np.lexsort((pick, pt.gid[pick], -pt.priority[pick].astype(np.int64)))]
        keep, closed = [], set()
        for p in pick.tolist():
            g = int(pt.gid[p])
            if gang and 0 <= g < G:
                if keep and int(pt.gid[keep[-1]]) == g:
                    keep.append(p)
                    continue
                if g in closed:
                    continue
                closed.add(g)
            keep.append(p)
        return np.array(keep, np.uint32)

    def broken_list(self, rule, gang):
        """A walk list that breaks one rule: "rising" (a priority above the one before), "twice" (a pod listed twice)
        or "split" (under gang, a group's preemptors around another pod of their priority)."""
        pt, G = self.model.pods, self.model.groups.n
        pods = self.walk_list(gang)
        if rule == "rising":
            d = np.flatnonzero(pt.priority[pods[:-1]] != pt.priority[pods[1:]])
            if len(d):
                i = int(d[0])
                pods[i], pods[i + 1] = pods[i + 1], pods[i]
                return pods
        if rule == "split":
            for g in range(G):
                for q in np.unique(pt.priority[pt.gid == g]):
                    mine = np.flatnonzero((pt.gid == g) & (pt.priority == q))
                    other = np.flatnonzero((pt.gid != g) & (pt.priority == q))
                    if len(mine) >= 2 and len(other):
                        return np.array([mine[0], other[0], mine[1]], np.uint32)
        return np.insert(pods, 1, pods[0]) if len(pods) else np.zeros(2, np.uint32)

    def preempt_walk(self, gang, rule=None):
        pods = self.walk_list(gang) if rule is None else self.broken_list(rule, gang)
        self.emit({"op": "preempt_walk", "pods": pods, "gang": gang, "rule": rule})

    def base(self, P=150, N=300, G=20):
        self.upload_nodes(N)
        self.upload_groups(G)
        self.upload_pods(P)
        self.all_sides()
        self.weights(on=True)
        self.round()

    # -- the scripted bursts --
    def r1(self):
        """Both persistent class indices past 4096 classes, then a small table that clears them, then a group row
        update whose new representative class is looked up in place in the cleared index."""
        self.upload_nodes(64)
        self.upload_groups(40)
        s = self.snap(5000, 1, 40)
        pt = s.pods
        pt.sel_mask = (self.rng.integers(0, 1 << 62, pt.n).astype(np.uint64) & np.uint64(~0xF & (2**64 - 1))) | \
            self.rng.integers(0, 16, pt.n).astype(np.uint64)
        pt.sel_mask[::5] = 0
        pt.tol_mask = self.rng.integers(0, 1 << 40, pt.n).astype(np.uint64)
        self.emit({"op": "upload_pods", "table": pt})
        self.all_sides()
        self.round("evaluate")
        self.upload_pods(60)
        self.all_sides()
        self.round()            # the groups' ids are assigned again in the cleared index
        self.update_groups("rep")
        self.round()            # ... so this update looks its new class up in place
        self.regimes.add("R1")

    def r2(self):
        for N in (0, 1, 511, 512, 513, 700, 64, 513, 0, 300):
            self.upload_nodes(N)
            self.all_sides()
            self.round()
        self.regimes.add("R2")

    def r3(self):
        self.upload_nodes(200)
        self._first = self.model.nodes
        self.all_sides()
        self.round()
        m = self.model
        # narrow -> scaled: a lane's values grow past the narrow limit in whole multiples of 2^20
        idx = np.arange(0, 200, 17, dtype=np.uint32)
        rows = m.nodes.take(idx).copy()
        rows.alloc[2] = (np.int64(1) << 40) + (np.arange(len(idx), dtype=np.int64) << 20)
        rows.requested[2] = 0
        self.emit({"op": "update_nodes", "idx": idx, "rows": rows, "mode": "scaled"})
        self.node_sides()
        self.round()
        rows = rows.copy()
        rows.alloc[2, 0] += 1   # an odd value: scaled -> wide
        self.emit({"op": "update_nodes", "idx": idx, "rows": rows, "mode": "wide"})
        self.node_sides()
        self.round()
        self.emit({"op": "update_nodes", "idx": idx, "rows": self._first.take(idx), "mode": "row back"})   # stays wide
        self.node_sides()
        self.round()
        s = self.snap(m.pods.n if m.pods is not None else 100, 1, m.groups.n if m.groups is not None else 10, aff=AFF)
        s.pods.req[2] = np.where(self.rng.random(s.pods.n) < 0.3, np.int64(1) << 41, 0)
        if m.groups is None:
            self.upload_groups(10)
        self.emit({"op": "upload_pods", "table": s.pods})   # a pod table that moves a scaled lane's unit
        self.all_sides()
        self.round()
        self.upload_nodes(200)   # a fresh table: narrow again
        self.all_sides()
        self.round()
        self.regimes.add("R3")

    def r4(self):
        self.base()
        self.round()
        m = self.model
        idx = np.array([0], np.uint32)
        owners = [("nz", "node", lambda: self.emit({"op": "update_nodes", "idx": idx, "rows": m.nodes.take(idx)})),
                  ("pref", "node", lambda: self.emit({"op": "update_nodes", "idx": idx, "rows": m.nodes.take(idx)})),
                  ("loc", "pod", lambda: self.emit({"op": "upload_pods", "table": m.pods})),
                  ("spread", "node", lambda: self.emit({"op": "upload_nodes", "table": m.nodes})),
                  ("ipa", "pod", lambda: self.emit({"op": "upload_pods", "table": m.pods}))]
        for name, half, drop in owners:
            drop()
            self.all_sides_but(name)
            self.round()            # BS_E_STATE while the weight is on (the non-zero columns: always)
            if name != "nz":
                self.emit({"op": "weights", **self._off(name)})
                self.round()        # the lists without the term
            self.side(name, "node")
            self.side(name, "pod")
            self.weights(on=True)
            self.round()            # the term back
        self.regimes.add("R4")

    def _off(self, name):
        return {"pref": {"pw": (0, 0)}, "loc": {"lw": (0, 0)}, "spread": {"w_spread": 0}, "ipa": {"w_ipa": 0}}[name]

    def all_sides_but(self, skip):
        """Every missing side but `skip` (a side's name, "ipf": the filter's halves and its placed side, "hp": the
        ports filter's halves, or "placed")."""
        m = self.model
        for name in ("nz", "pref", "loc", "spread", "ipa"):
            if name == skip:
                continue
            for half in ("node", "pod"):
                if m.side[name + "_" + half] is None:
                    self.side(name, half)
        for half in ("node", "pod"):
            if skip != "ipf" and getattr(m, "ipf_" + half) is None:
                self.ipf(half)
            if skip != "hp" and getattr(m, "hp_" + half) is None:
                self.hp(half)
        if skip not in ("ipf", "placed") and m.ipf_placed is None:
            self.placed()

    def r5(self):
        self.base()
        m = self.model
        bad = m.nodes.copy()
        if bad.n:
            bad.requested[0, bad.n // 2] = LIMIT + 1
        else:
            bad = self.snap(1, 5, 1).nodes
            bad.alloc[1, 2] = -LIMIT - 1
        self.emit({"op": "upload_nodes", "table": bad})
        self.round()                 # BS_E_STATE, never a round on the previous snapshot
        self.emit({"op": "update_nodes", "idx": np.zeros(1, np.uint32), "rows": bad.take([0])})
        self.upload_nodes(250)
        self.all_sides()
        self.round()
        bad = m.groups.copy()
        bad.min_res[0, 0] = -(LIMIT + 1)
        self.emit({"op": "upload_groups", "table": bad})
        self.round()
        self.upload_groups(12)
        bad = m.pods.copy()
        bad.req[1, -1] = LIMIT + 1
        self.emit({"op": "upload_pods", "table": bad})
        self.round()
        self.upload_pods(100)
        self.all_sides()
        self.round()
        self.regimes.add("R5")

    def r6(self):
        self.upload_nodes(0)
        self.upload_groups(10)
        self.upload_pods(80)
        self.all_sides()
        self.weights(on=True)
        self.round()
        self.upload_nodes(130)
        self.upload_groups(0)
        self.upload_pods(0)
        self.all_sides()
        self.round()
        self.upload_groups(7)
        self.upload_pods(90)
        self.all_sides()
        self.round()
        self.regimes.add("R6")

    def r7(self):
        """The filter's lifecycle: each half dropped by the call that owns it and uploaded again, a node table of
        another size, a pod table refused for its lane count, a failing pod half, and the four refusals."""
        self.upload_nodes(300)
        self.upload_groups(20)
        self.upload_pods(150)
        self.all_sides_but("ipf")
        self.weights(on=True)
        self.switch(True)
        self.round()                 # BS_E_STATE: no halves
        self.ipf("node")
        self.ipf("pod")
        self.round()
        self.update_nodes(str(self.rng.choice(["widen", "flags", "labels"])))
        self.all_sides_but("ipf")
        self.round()                 # BS_E_STATE: the node half went with the update
        self.ipf("node")
        self.round()
        self.upload_nodes(int(self.rng.choice([513, 700])))   # another Npad for the pass planes
        self.all_sides()
        self.round()
        lanes = random_snapshot(self._k(), P=40, N=1, G=1, L=self.L + 1).pods
        self.emit({"op": "upload_pods", "table": lanes})   # BS_E_INVAL: the pod table stays, its sides go
        self.all_sides_but("ipf")
        self.round()                 # BS_E_STATE: the pod half went with the refused call
        self.ipf("pod")
        self.round()
        self.ipf("pod", bad=True)    # BS_E_INDEX
        self.round()                 # BS_E_STATE
        self.ipf("pod")
        self.round()
        self.bound()
        for kind in ("first_fit", "priority"):
            self.emit({"op": "replay", "priority": kind == "priority"})   # BS_E_INVAL while the filter is on
        self.emit({"op": "preempt", "pods": np.arange(min(self.model.pods.n, 40), dtype=np.uint32)})
        self.preempt_walk(False)
        self.switch(False)
        self.emit({"op": "replay", "priority": False})
        self.emit({"op": "preempt", "pods": np.arange(min(self.model.pods.n, 40), dtype=np.uint32)})
        self.preempt_walk(True)
        self.switch(True)
        self.round()
        self.regimes.add("R7")

    def r8(self):
        """More than 4096 fit classes under the filter, and pod halves that put the pods in new filter classes at
        every round until compact_fit_index rebuilds the fit index, with the switch toggled, a group row update and a
        new affinity table in between; then a small pod table with the switch off and on."""
        self.upload_nodes(64)
        self.upload_groups(40)
        pt = self.snap(R8_PODS, 1, 40).pods
        pt.tol_mask = self.rng.integers(0, 1 << 62, pt.n).astype(np.uint64)   # a fit class per pod
        self.emit({"op": "upload_pods", "table": pt})
        self.all_sides()
        self.switch(True)
        self.round("evaluate")
        for k in range(R8_ROUNDS):
            self.ipf("pod", spread=R8_SPREAD)
            if k % 4 == 1:
                self.switch(False)
                self.round()
                self.switch(True)
            if k == R8_ROUNDS // 2:
                self.update_groups("rep")
                self.emit({"op": "upload_affinity", "bits": self.snap(1, 64, 1, aff=AFF).aff_bits})
            self.round()
        self.upload_pods(50)
        self.all_sides()
        self.switch(False)
        self.round()
        self.switch(True)
        self.round()
        self.regimes.add("R8")

    def r9(self):
        """Preemption with PodDisruptionBudget bits and the walk: after a group row update (the bound table stays),
        after a node row update and after a group upload (both drop it), and one walk per broken list rule."""
        self.switch(False)
        self.hp_switch(False)
        self.base()
        self.bound()
        self.walk("preempt")
        self.preempt_walk(False)
        self.preempt_walk(True)
        self.update_groups("creation")
        self.emit({"op": "preempt", "pods": np.arange(min(self.model.pods.n, 40), dtype=np.uint32)})
        self.update_nodes(str(self.rng.choice(["widen", "flags", "labels"])))
        self.preempt_walk(False)     # BS_E_STATE: the update dropped the bound table
        self.bound()
        self.preempt_walk(bool(self.rng.random() < 0.5))
        self.upload_groups(self.model.groups.n)
        self.preempt_walk(True, "split")   # BS_E_STATE: the state checks come before the list rules
        self.bound()
        for rule, gang in (("rising", False), ("twice", False), ("split", True)):
            self.preempt_walk(gang, rule)
        self.preempt_walk(True)
        self.regimes.add("R9")

    def r10(self):
        """The ports filter's lifecycle: the switch without halves, each half dropped by the call that owns it, a node
        table of another size, a pod table refused for its lane count followed by a want half other than the one before
        and a round (the pods' fit classes are built again from their base classes, not from the classes the filter
        gave them), each failing node half, a dictionary that the want bits pass, preemption refused, the switch off."""
        self.upload_nodes(300)
        self.upload_groups(20)
        self.upload_pods(150)
        self.all_sides_but("hp")
        self.weights(on=True)
        self.switch(False)
        self.hp_switch(True)
        self.round()                 # BS_E_STATE: no halves
        self.hp("node")
        self.round()                 # BS_E_STATE: no pod half
        self.hp("pod")
        self.round()
        self.update_nodes(str(self.rng.choice(["widen", "flags", "labels"])))
        self.all_sides_but("hp")
        self.round()                 # BS_E_STATE: the node half went with the update
        self.hp("node")
        self.round()
        self.upload_pods(150)
        self.all_sides_but("hp")
        self.round()                 # BS_E_STATE: the pod half went with the pod table
        self.hp("pod")
        self.round()
        self.upload_nodes(int(self.rng.choice([513, 700])))   # another Npad
        self.all_sides()
        self.round()
        lanes = random_snapshot(self._k(), P=40, N=1, G=1, L=self.L + 1).pods
        self.emit({"op": "upload_pods", "table": lanes})   # BS_E_INVAL: the pod table stays, its sides go
        self.all_sides_but("hp")
        self.round()                 # BS_E_STATE: the pod half went with the refused call
        self.emit({"op": "hp", "half": "pod", "n": self.model.pods.n, "cols": np.zeros(self.model.pods.n, np.uint64)})
        self.round()                 # no pod wants a port: every node passes the filter
        self.hp("pod")
        self.round()
        for bad in ("port", "twice", "used", "many"):
            self.hp("node", bad=bad)     # BS_E_RANGE, BS_E_INVAL, BS_E_INDEX, BS_E_INVAL
        self.hp("node", wrong_len=True)  # BS_E_INVAL
        self.round()                 # BS_E_STATE
        self.hp("pod", wrong_len=True)
        self.hp("node", n_entries=3)
        self.round()                 # BS_E_STATE: the pod half failed
        self.hp("pod")
        self.round()                 # BS_E_INDEX: want bits past the 3 entries
        self.hp("node")
        self.round()
        self.bound()
        self.emit({"op": "preempt", "pods": np.arange(min(self.model.pods.n, 40), dtype=np.uint32)})   # BS_E_INVAL
        self.preempt_walk(False)     # BS_E_INVAL
        self.hp_switch(False)
        self.round()
        self.regimes.add("R10")

    def r11(self):
        """More than 4096 fit classes under the ports filter, and want halves that put every pod in a new conflict
        class at each round until compact_fit_index rebuilds the fit index; the inter-pod switch toggled in between and
        a group row update; then a small pod table.  The dictionary's entries have distinct ports, so each entry
        conflicts with itself alone and a pod's conflict mask is its want mask."""
        self.upload_nodes(64)
        self.upload_groups(40)
        pt = self.snap(R8_PODS, 1, 40).pods
        pt.tol_mask = self.rng.integers(0, 1 << 62, pt.n).astype(np.uint64)   # a fit class per pod
        self.emit({"op": "upload_pods", "table": pt})
        self.all_sides_but("hp")
        K = R11_ENTRIES
        entries = np.array([(1 + k % 2, k % 2, 2000 + k) for k in range(K)], np.int64)
        used = np.bitwise_or.reduce(self._bits(self.model.nodes.n, K, 0.04), axis=1)
        self.emit({"op": "hp", "half": "node", "n": len(used), "cols": (entries, used)})
        self.switch(True)
        self.hp_switch(True)
        for k in range(R11_ROUNDS):
            want = np.bitwise_or.reduce(self._bits(pt.n, K, 0.06), axis=1)
            self.emit({"op": "hp", "half": "pod", "n": pt.n, "cols": want})
            if k % 3 == 1:
                self.switch(not self.model.ipf_on)
            if k == R11_ROUNDS // 2:
                self.update_groups("rep")
            self.round("evaluate" if k == 0 else None)
        self.upload_pods(50)
        self.all_sides()
        self.round()
        self.switch(False)
        self.round()
        self.regimes.add("R11")

    def _bits(self, n, K, p):
        """[n, K] uint64: bit k of column k with probability p."""
        return np.where(self.rng.random((n, K)) < p, np.uint64(1) << np.arange(K, dtype=np.uint64), np.uint64(0))

    def r12(self):
        """Walks under the inter-pod filter, the ports filter and both: right after a new filter half and before any
        round (the walk runs the filter's pre-pass for the next evaluation), after bs_update_nodes and the node halves
        again; a refused pod upload drops the placed side, a placed term past the node half's dictionary, and with the
        filter off the placed side is not read."""
        self.upload_nodes(300)
        self.upload_groups(20)
        self.upload_pods(150)
        self.all_sides()
        self.weights(on=True)
        self.walk_weights()
        for on in ("ipf", "hp", "both"):
            self.switch(on != "hp")
            self.hp_switch(on != "ipf")
            self.round()
            if on != "hp":
                self.ipf("node")
            if on != "ipf":
                self.hp("node")
            for kind in ("first_fit", "priority"):
                self.walk(kind)
            self.round()
            self.update_nodes(str(self.rng.choice(["widen", "flags", "labels"])))
            self.node_sides()
            for kind in ("first_fit", "priority"):
                self.walk(kind)
            self.round()
        lanes = random_snapshot(self._k(), P=40, N=1, G=1, L=self.L + 1).pods
        self.emit({"op": "upload_pods", "table": lanes})   # BS_E_INVAL: the placed side goes with the pod sides
        self.all_sides_but("placed")
        self.walk("first_fit")       # BS_E_INVAL: the filter is on without the placed side
        self.placed()
        self.walk("priority")
        self.placed(bad="term")
        self.walk("first_fit")       # BS_E_INDEX: a placed term past the node half's dictionary
        self.placed(bad="class")     # BS_E_INDEX
        self.placed(bad="own")       # BS_E_RANGE
        self.placed(bad="term")
        self.switch(False)
        self.walk("priority")        # the placed side is not read
        self.hp_switch(False)
        self.walk("first_fit")
        self.switch(True)
        self.placed()
        self.round()
        self.regimes.add("R12")

    # -- random ops --
    def ports_or_walk_op(self):
        m = self.model
        r = self.rng.random()
        if r < 0.2:
            self.hp_switch(not m.hp_on)
            self.round()
        elif r < 0.45:
            if self.rng.random() < 0.3:
                self.hp_seed = self._k()   # new halves: the pod half first, then the node half
                self.hp("pod")
                self.hp("node")
            else:
                half = str(self.rng.choice(["node", "pod"]))
                bad = self.rng.choice([None, "port", "twice", "used", "many"]) if self.rng.random() < 0.15 else None
                self.hp(half, wrong_len=self.rng.random() < 0.1, bad=bad,
                        n_entries=3 if self.rng.random() < 0.1 else 12)
            self.round()
        elif r < 0.6:
            bad = self.rng.choice([None, "class", "own", "term"]) if self.rng.random() < 0.2 else None
            self.placed(wrong_len=self.rng.random() < 0.1, bad=bad)
            self.walk(str(self.rng.choice(["first_fit", "priority"])))
        else:
            on = str(self.rng.choice(["ipf", "hp", "both"]))
            self.switch(on != "hp")
            self.hp_switch(on != "ipf")
            if m.ipf_placed is None and self.rng.random() < 0.8:
                self.placed()
            if self.rng.random() < 0.5:
                self.walk_weights()
            self.walk(str(self.rng.choice(["first_fit", "priority"])))

    def filter_or_preempt_op(self):
        m = self.model
        r = self.rng.random()
        if r < 0.25:
            self.switch(not m.ipf_on)
            self.round()
        elif r < 0.5:
            if self.rng.random() < 0.3:
                self.ipf_seed = self._k()   # new halves: the pod half first, then the node half
                self.ipf("pod")
                self.ipf("node")
            else:
                self.ipf(str(self.rng.choice(["node", "pod"])), wrong_len=self.rng.random() < 0.2,
                         mismatch=self.rng.random() < 0.1)
            self.round()
        elif r < 0.65:
            self.bound()
            self.walk("preempt")
        else:
            if m.bound is None or self.rng.random() < 0.4:
                self.bound()
            gang = bool(self.rng.random() < 0.5)
            rule = str(self.rng.choice(["rising", "twice", "split"])) if self.rng.random() < 0.2 else None
            self.preempt_walk(gang, rule)

    def random_op(self):
        m = self.model
        r = self.rng.random()
        if m.nodes is None or m.pods is None or m.groups is None:
            self.base()
        elif r < 0.10:
            self.filter_or_preempt_op()
        elif r < 0.17:
            self.ports_or_walk_op()
        elif r < 0.23:   # without its affinity table now and then: the pods' classes are BS_E_INDEX until it comes
            self.upload_nodes(int(self.rng.choice([1, 33, 511, 512, 513, 900])), aff=AFF if self.rng.random() < 0.85 else 0)
            self.all_sides(("node",))
        elif r < 0.29:
            self.upload_pods(int(self.rng.choice([0, 1, 70, self.max_p + 13])), aff=AFF if self.rng.random() < 0.8 else 0)
            self.all_sides(("pod",))
        elif r < 0.32:
            self.upload_groups(int(self.rng.choice([0, 1, 9, 31])), aff=AFF if self.rng.random() < 0.8 else 0)
        elif r < 0.42 and m.nodes.n:
            self.update_nodes(str(self.rng.choice(["widen", "back", "flags", "labels"])))
            if self.rng.random() < 0.85:   # else the next rounds answer BS_E_STATE until a side op brings them back
                self.node_sides()
                self.round()
        elif r < 0.48 and m.groups.n:
            self.update_groups(str(self.rng.choice(["rep", "creation"])))
            self.round()
        elif r < 0.55:   # a new table (the nodes' class fits change), or none (the pods' classes are out of range)
            bits = self.snap(1, m.nodes.n, 1, aff=AFF).aff_bits if self.rng.random() < 0.75 else None
            self.emit({"op": "upload_affinity", "bits": bits})
            self.round()
        elif r < 0.65:
            name = str(self.rng.choice(["nz", "pref", "loc", "spread", "ipa"]))
            half = str(self.rng.choice(["node", "pod"]))
            self.side(name, half, mismatch=self.rng.random() < 0.3, wrong_len=self.rng.random() < 0.1)
        elif r < 0.72:
            self.weights(on=bool(self.rng.random() < 0.6))
        elif r < 0.78:
            kind = str(self.rng.choice(["nodes", "groups", "pods", "index", "lanes"]))
            if kind == "index" and m.nodes.n:
                self.emit({"op": "update_nodes", "idx": np.array([m.nodes.n], np.uint32), "rows": m.nodes.take([0])})
            elif kind == "groups":
                bad = m.groups.copy()
                if bad.n:
                    bad.min_res[1, -1] = LIMIT + 1
                self.emit({"op": "upload_groups", "table": bad})
            elif kind == "pods" and m.pods.n:
                bad = m.pods.copy()
                bad.req[0, 0] = -(LIMIT + 1)
                self.emit({"op": "upload_pods", "table": bad})
            elif kind == "lanes":   # refused for its lane count: the pod table stays, its sides go
                self.emit({"op": "upload_pods", "table": random_snapshot(self._k(), P=20, N=1, G=1, L=self.L + 1).pods})
        elif r < 0.85:
            self.walk(str(self.rng.choice(["first_fit", "priority", "preempt"])))
        else:
            self.round()


BURSTS = ("r1", "r2", "r3", "r4", "r5", "r6", "r7", "r8", "r9", "r10", "r11", "r12")
R8_PODS, R8_ROUNDS, R8_SPREAD = 4200, 9, 64
R11_ENTRIES, R11_ROUNDS = 40, 10


def generate(seed, n_ops=30, lanes=None):
    """(ops, regimes): about n_ops random ops around one scripted burst (seed % len(BURSTS) picks it; seeds >= 6 add
    another), every op as the dict Model.apply takes; regimes names the bursts the sequence ran."""
    g = Generator(seed, lanes or [5, 6, 9][seed % 3])
    n = len(BURSTS)
    bursts = [BURSTS[seed % n]] + ([BURSTS[(seed + 4) % n]] if seed >= 6 else [])
    at = sorted(int(x) for x in g.rng.integers(0, n_ops, len(bursts)))
    g.base()
    for i in range(n_ops):
        while at and at[0] == i:
            getattr(g, bursts.pop(0))()
            at.pop(0)
        g.random_op()
    g.round()
    return g.ops, g.regimes, g.L
