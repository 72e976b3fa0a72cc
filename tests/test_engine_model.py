"""CPU: the host model of a long-lived engine (tests/engine_model.py) and its op generator, without a device: row
updates through the model equal the tables built directly, the generator is deterministic and reaches every scripted
regime across the seeds the GPU test runs, and the model's expected outputs come from the restatements on a short
sequence (which keeps the reference side honest and bounds its cost).  The drop rules, check orders and refusals of
the MatchInterPodAffinity filter, its placed side and the PodFitsHostPorts filter, the preemption walk's list rules,
and the invariants of a round under the filter are pinned on hand-built op lists; the walk references the model picks
agree with each other wherever more than one applies."""
import functools
import operator

import numpy as np

import engine_model as em
import host_ports_ref as hr
import interpod_filter_ref as fr
import interpod_walk_ref as iwr
import locality_priority_ref as lpr
from oracle import oracle
from randsnap import S, random_snapshot

SEEDS = range(len(em.BURSTS))   # the GPU test's seeds


def _same(a, b):
    for f in a.__dataclass_fields__:
        x, y = getattr(a, f), getattr(b, f)
        assert (x is None) == (y is None), f
        if x is not None:
            np.testing.assert_array_equal(x, y, err_msg=f)


def test_row_updates_equal_tables_built_directly():
    snap = random_snapshot(11, P=40, N=90, G=25, L=6)
    other = random_snapshot(12, P=40, N=90, G=25, L=6)
    m = em.Model(6)
    assert m.apply({"op": "upload_nodes", "table": snap.nodes}) is None
    assert m.apply({"op": "upload_groups", "table": snap.groups}) is None
    nodes, groups = snap.nodes.copy(), snap.groups.copy()
    for k, idx in enumerate([np.array([0, 5, 89]), np.arange(0, 90, 7), np.array([44])]):
        idx = idx.astype(np.uint32)
        assert m.apply({"op": "update_nodes", "idx": idx, "rows": other.nodes.take(idx)}) is None
        nodes.alloc[:, idx], nodes.requested[:, idx] = other.nodes.alloc[:, idx], other.nodes.requested[:, idx]
        for f in ("pod_count", "alloc_present", "req_present", "label_mask", "taint_mask", "flags"):
            getattr(nodes, f)[idx] = getattr(other.nodes, f)[idx]
        _same(m.nodes, nodes)
        assert len(m.history) == k + 1
        gidx = idx[idx < 25]
        assert m.apply({"op": "update_groups", "idx": gidx, "rows": other.groups.take(gidx)}) is None
        groups.min_res[:, gidx] = other.groups.min_res[:, gidx]
        for f in ("min_member", "scheduled", "matched", "flags", "min_res_present", "rep_sel", "rep_tol", "creation_ns",
                  "name_rank"):
            getattr(groups, f)[gidx] = getattr(other.groups, f)[gidx]
        _same(m.groups, groups)
    _same(snap.nodes, random_snapshot(11, P=40, N=90, G=25, L=6).nodes)   # the uploaded table was not written
    # failing updates leave every row, and an index past the table is BS_E_INDEX
    bad = other.nodes.take([1]).copy()
    bad.alloc[0, 0] = em.LIMIT + 1
    assert m.apply({"op": "update_nodes", "idx": np.array([3], np.uint32), "rows": bad}) == em.E_RANGE
    assert m.apply({"op": "update_nodes", "idx": np.array([90], np.uint32), "rows": other.nodes.take([1])}) == em.E_INDEX
    assert m.apply({"op": "update_groups", "idx": np.array([25], np.uint32), "rows": other.groups.take([1])}) == em.E_INDEX
    _same(m.nodes, nodes)
    _same(m.groups, groups)


def test_drop_rules_and_check_order():
    snap = random_snapshot(13, P=30, N=50, G=6, L=5, aff=2)
    m = em.Model(5)
    assert m.apply({"op": "evaluate", "priority": True}) == em.E_STATE
    for op in ({"op": "upload_nodes", "table": snap.nodes}, {"op": "upload_affinity", "bits": snap.aff_bits},
               {"op": "upload_groups", "table": snap.groups}, {"op": "upload_pods", "table": snap.pods}):
        assert m.apply(op) is None
    nz = S.nonzero_requests(snap, 1)
    for half, cols in (("node", nz[0]), ("pod", nz[1])):
        assert m.apply({"op": "side", "name": "nz", "half": half, "n": cols.shape[1], "cols": cols}) is None
    assert m.apply({"op": "evaluate", "priority": True}) is None
    assert m.apply({"op": "weights", "w_spread": 1}) is None
    assert m.apply({"op": "evaluate", "priority": True}) == em.E_STATE
    assert m.apply({"op": "replay", "priority": True}) == em.E_INVAL      # refused before the tables are looked at
    assert m.apply({"op": "weights", "w_spread": 0}) is None
    bad = snap.nodes.copy()
    bad.alloc[1, 3] = -(em.LIMIT + 1)
    assert m.apply({"op": "upload_nodes", "table": bad}) == em.E_RANGE   # the old snapshot goes with it
    assert m.nodes is None and m.aff is None and m.side["nz_node"] is None and m.side["nz_pod"] is not None
    assert m.apply({"op": "evaluate", "priority": True}) == em.E_STATE
    assert m.apply({"op": "upload_nodes", "table": snap.nodes}) is None
    assert m.apply({"op": "side", "name": "nz", "half": "node", "n": 50, "cols": nz[0]}) is None
    assert m.apply({"op": "evaluate", "priority": True}) == em.E_INDEX    # the pods name classes the table lacks
    assert m.apply({"op": "side", "name": "nz", "half": "node", "n": 51, "cols": nz[0]}) == em.E_INVAL
    assert m.side["nz_node"] is None


def test_generator_is_deterministic_and_reaches_every_regime():
    seen = set()
    for seed in SEEDS:
        ops, regimes, L = em.generate(seed)
        again, regimes2, _ = em.generate(seed)
        assert regimes == regimes2 and regimes
        assert [em.describe(o) for o in ops] == [em.describe(o) for o in again]
        seen |= regimes
        kinds = {o["op"] for o in ops}
        assert {"upload_nodes", "upload_pods", "upload_groups", "side", "weights", "evaluate"} <= kinds
    assert seen == {f"R{k}" for k in range(1, len(em.BURSTS) + 1)}
    assert {em.BURSTS[s % len(em.BURSTS)] for s in SEEDS} == set(em.BURSTS)   # each burst runs first in some seed


def test_sequences_reach_the_edges():
    """Across the seeds: N, P and G of 0, node counts on both sides of the 512-node tile, the class indices past
    4096, every side refused once (wrong length), every error the model predicts, and a round after each."""
    codes, sizes, P_max, by_op = set(), set(), 0, {}
    for seed in SEEDS:
        ops, _, L = em.generate(seed)
        m = em.Model(L)
        for op in ops:
            rc = m.apply(op)
            codes.add(rc)
            by_op.setdefault(op["op"], set()).add(rc)
            if op["op"] == "upload_nodes":
                sizes.add(op["table"].n)
            if op["op"] == "upload_pods":
                sizes.add(("P", op["table"].n))
                P_max = max(P_max, op["table"].n)
            if op["op"] == "upload_groups":
                sizes.add(("G", op["table"].n))
    assert {None, em.E_STATE, em.E_RANGE, em.E_INDEX, em.E_INVAL} <= codes
    # every refusal of the ports filter's node half and of the placed side, and the walks' own ones
    assert {None, em.E_INVAL, em.E_RANGE, em.E_INDEX} <= by_op["hp"], by_op["hp"]
    assert {None, em.E_INDEX, em.E_RANGE} <= by_op["placed"], by_op["placed"]
    assert {None, em.E_INVAL, em.E_INDEX} <= by_op["replay"], by_op["replay"]
    assert {None, em.E_STATE, em.E_INDEX} <= by_op["evaluate"]
    assert {0, 1, 511, 512, 513, ("P", 0), ("G", 0)} <= sizes
    assert P_max >= 4097


def test_expect_on_a_short_sequence():
    ops, _, L = em.generate(5, n_ops=6)
    m = em.Model(L)
    cfgs = (dict(score=True, fit_bitmap=True, filter=True, reasons=True, priority_k=8),
            dict(topk=8, priority_k=8, reasons=True))
    rounds = 0
    for op in ops[:60]:
        if m.apply(op) is None and op["op"] == "evaluate":
            for cfg in cfgs:
                out = m.expect(cfg)
                P, N = m.pods.n, m.nodes.n
                assert out["prefilter"].shape == (P,)
                assert out["priority_nodes"].shape == (P, 8)
                fits = (out["priority_nodes"] >= 0).sum(axis=1)
                np.testing.assert_array_equal(fits, np.minimum(8, out["feasible_count"]))
                if "topk_nodes" in out:
                    np.testing.assert_array_equal(out["topk_nodes"][:, 0], np.where(out["feasible_count"] > 0,
                                                                                     out["best_node"], -1))
                if "reason_rows" in out:
                    assert out["reason_rows"].shape == (P, 4 + L)
                assert len(out["lanes"][0]) == L
            rounds += 1
    assert rounds >= 2


def test_row_updates_and_affinity_reach_compared_rounds():
    """Each kind of node row update (a lane widened, a row put back, flags, labels, and R3's narrow -> scaled -> wide
    -> row back) is followed by a successful round before the next full node upload, and many successful rounds have
    pods and groups naming affinity classes, some right after a new affinity table: the GPU test compares those rounds
    with the references, so these states are checked and not only refused."""
    reached, aff_rounds, fresh_aff, group_aff = set(), 0, 0, 0
    for seed in SEEDS:
        ops, _, L = em.generate(seed)
        m = em.Model(L)
        pending, new_table = set(), False
        for op in ops:
            rc = m.apply(op)
            if op["op"] == "upload_nodes":
                pending = set()
            elif op["op"] == "update_nodes" and rc is None and "mode" in op:
                pending.add(op["mode"])
            elif op["op"] == "upload_affinity" and rc is None:
                new_table = op["bits"] is not None
            elif op["op"] == "evaluate" and rc is None:
                reached |= pending
                pending = set()
                if m.pods.aff_class is not None and (m.pods.aff_class != S.AFF_NONE).any():
                    aff_rounds += 1
                    fresh_aff += new_table
                group_aff += m.groups.rep_aff is not None and bool((m.groups.rep_aff != S.AFF_NONE).any())
                new_table = False
    assert reached == {"widen", "back", "flags", "labels", "scaled", "wide", "row back"}
    assert aff_rounds >= 50 and fresh_aff >= 20 and group_aff >= 50, (aff_rounds, fresh_aff, group_aff)


def test_r1_updates_a_group_in_place_after_the_indices_cleared():
    """R1 runs a round between the upload that clears both class indices and the group row update, so the update
    finds the groups' ids current and looks its new representative class up in place in the cleared index."""
    g = em.Generator(0, 5)
    g.base()
    g.r1()
    kinds = [o["op"] for o in g.ops]
    at = len(kinds) - 1 - kinds[::-1].index("update_groups")
    assert kinds[at + 1] == "evaluate"
    before = kinds[:at]
    last_pods = len(before) - 1 - before[::-1].index("upload_pods")
    assert "evaluate" in before[last_pods:]
    assert g.ops[last_pods]["table"].n < 4096 // 4


def _loaded(seed=21, P=60, N=90, G=12, L=5):
    """A model with every table, the non-zero columns and both filter halves of one cluster; the switch off."""
    snap = random_snapshot(seed, P=P, N=N, G=G, L=L, aff=2)
    m = em.Model(L)
    for op in ({"op": "upload_nodes", "table": snap.nodes}, {"op": "upload_affinity", "bits": snap.aff_bits},
               {"op": "upload_groups", "table": snap.groups}, {"op": "upload_pods", "table": snap.pods}):
        assert m.apply(op) is None
    nz = S.nonzero_requests(snap, 1)
    for half, cols in (("node", nz[0]), ("pod", nz[1])):
        assert m.apply({"op": "side", "name": "nz", "half": half, "n": cols.shape[1], "cols": cols}) is None
    node, pods = S.node_interpod_filter(snap, 3)
    assert m.apply({"op": "ipf", "half": "node", "n": N, "cols": node}) is None
    assert m.apply({"op": "ipf", "half": "pod", "n": P, "cols": pods}) is None
    return m, snap, node, pods


def test_filter_drop_rules_and_check_order():
    m, snap, node, pods = _loaded()
    ev = {"op": "evaluate", "priority": True}
    half = lambda h, cols, n=None: {"op": "ipf", "half": h, "cols": cols,
                                    "n": (snap.nodes.n if h == "node" else snap.pods.n) if n is None else n}
    assert m.apply(ev) is None and not m.ipf_round
    assert m.apply({"op": "ipf_switch", "on": True}) is None
    assert m.apply(ev) is None and m.ipf_round
    # bs_update_nodes drops the node half, also a call that changes no row or fails
    for idx, rows in ((np.zeros(0, np.uint32), snap.nodes.take(np.zeros(0, np.int64))), (np.array([snap.nodes.n], np.uint32),
                                                                      snap.nodes.take([0]))):
        m.apply({"op": "update_nodes", "idx": idx, "rows": rows})
        assert m.ipf_node is None and m.ipf_pod is not None
        assert m.apply(half("node", node)) is None
    assert m.apply({"op": "update_nodes", "idx": np.array([1], np.uint32), "rows": snap.nodes.take([1])}) is None
    assert m.apply({"op": "side", "name": "nz", "half": "node", "n": snap.nodes.n,
                    "cols": S.nonzero_requests(snap, 1)[0]}) is None
    assert m.apply(ev) == em.E_STATE            # the filter's half, after the priority sides are back
    assert m.apply(half("node", node)) is None
    assert m.apply(ev) is None
    # bs_upload_nodes drops it, also one that fails validation
    bad = snap.nodes.copy()
    bad.alloc[0, 0] = em.LIMIT + 1
    assert m.apply({"op": "upload_nodes", "table": bad}) == em.E_RANGE
    assert m.ipf_node is None
    assert m.apply(half("node", node)) == em.E_STATE    # without its table
    assert m.apply({"op": "upload_nodes", "table": snap.nodes}) is None
    assert m.apply({"op": "upload_affinity", "bits": snap.aff_bits}) is None
    assert m.apply({"op": "side", "name": "nz", "half": "node", "n": snap.nodes.n,
                    "cols": S.nonzero_requests(snap, 1)[0]}) is None
    wide = (node[0], np.concatenate([node[1], node[1][:, :1]], axis=1), *node[2:])
    assert m.apply(half("node", wide, snap.nodes.n + 1)) == em.E_INVAL and m.ipf_node is None
    off_table = (*node[:3], np.r_[node[3][:-1], np.uint32(snap.nodes.n)], *node[4:])
    assert m.apply(half("node", off_table)) == em.E_INDEX and m.ipf_node is None   # a bound pod on no node
    assert m.apply(half("node", node)) is None
    # bs_upload_pods drops the pod half, also a call refused for its lane count (which keeps the pod table)
    other = random_snapshot(5, P=7, N=1, G=1, L=6).pods
    assert m.apply({"op": "upload_pods", "table": other}) == em.E_INVAL
    assert m.pods is snap.pods and m.ipf_pod is None and m.side["nz_pod"] is None
    assert m.apply({"op": "side", "name": "nz", "half": "pod", "n": snap.pods.n,
                    "cols": S.nonzero_requests(snap, 1)[1]}) is None
    assert m.apply(ev) == em.E_STATE
    # a failing half leaves it dropped: a pod class out of range is BS_E_INDEX, a wrong length BS_E_INVAL
    pcls, cl = pods
    assert m.apply(half("pod", (np.full(len(pcls), len(cl[0]) - 1, np.uint32), cl))) == em.E_INDEX
    assert m.apply(half("pod", (pcls[:-1], cl), snap.pods.n - 1)) == em.E_INVAL
    assert m.ipf_pod is None and m.apply(ev) == em.E_STATE
    # a term outside the node half's dictionary is BS_E_INDEX at evaluation, after the priority sides' checks
    far = (pcls, (cl[0], np.full_like(cl[1], len(node[2])), cl[2], cl[3]))
    assert m.apply(half("pod", far)) is None
    assert m.apply(ev) == em.E_INDEX
    assert m.apply({"op": "weights", "w_spread": 1}) is None
    assert m.apply(ev) == em.E_STATE            # the spread sides are checked first
    assert m.apply({"op": "weights", "w_spread": 0}) is None
    assert m.apply(half("pod", pods)) is None
    assert m.apply(ev) is None
    # ... and before the affinity ids
    assert m.apply({"op": "upload_affinity", "bits": None}) is None
    assert m.apply({"op": "ipf", "half": "pod", "n": snap.pods.n, "cols": far}) is None
    assert m.apply(ev) == em.E_INDEX
    assert m.apply(half("pod", pods)) is None
    assert m.apply(ev) == em.E_INDEX            # now the affinity ids
    assert m.apply({"op": "ipf_switch", "on": False}) is None
    assert m.apply(ev) == em.E_INDEX and m.ipf_round


def test_refusals_and_walk_rules():
    m, snap, node, pods = _loaded()
    pt = snap.pods
    walk = lambda p, gang=False: {"op": "preempt_walk", "pods": np.asarray(p, np.uint32), "gang": gang}
    refusals = ({"op": "replay", "priority": False}, {"op": "replay", "priority": True},
                {"op": "preempt", "pods": np.arange(5, dtype=np.uint32)}, walk([0]))
    assert m.apply({"op": "ipf_switch", "on": True}) is None
    for op in refusals:   # before every other check: there is no bound table yet, and a broken list
        assert m.apply(op) == em.E_INVAL
    assert m.apply(walk([0, 0])) == em.E_INVAL
    assert m.apply({"op": "ipf_switch", "on": False}) is None
    assert m.apply(refusals[0]) is None
    assert m.apply(refusals[2]) == em.E_STATE and m.apply(refusals[3]) == em.E_STATE
    assert m.apply(walk([0, 0])) == em.E_STATE   # the state checks come before the list rules
    assert m.apply({"op": "upload_bound", "table": S.bound_pods(snap, 2, max_per_node=4, violating=0.3)}) is None
    assert m.apply(walk([pt.n])) == em.E_INDEX
    order = np.lexsort((np.arange(pt.n), pt.gid, -pt.priority.astype(np.int64)))
    assert m.apply(walk(order[:20])) is None
    assert m.apply(walk(order[:20][::-1])) == em.E_INVAL                         # rising priorities
    assert m.apply(walk(np.r_[order[:5], order[4]])) == em.E_INVAL               # a pod twice
    # a group split around another pod of its priority: a rule under gang only; gids >= n_groups are units of one
    g, q = next((g, q) for g in range(snap.groups.n) for q in np.unique(pt.priority[pt.gid == g])
                if ((pt.gid == g) & (pt.priority == q)).sum() >= 2 and ((pt.gid != g) & (pt.priority == q)).any())
    a, b = np.flatnonzero((pt.gid == g) & (pt.priority == q))[:2]
    h = np.flatnonzero((pt.gid != g) & (pt.priority == q))[0]
    assert m.apply(walk([a, h, b])) is None
    assert m.apply(walk([a, h, b], gang=True)) == em.E_INVAL
    far = pt.copy()
    far.gid[[a, b]] = snap.groups.n + 3
    far.gid[h] = snap.groups.n + 4
    assert m.apply({"op": "upload_pods", "table": far}) is None
    assert m.apply({"op": "upload_bound", "table": S.bound_pods(snap, 2, max_per_node=4)}) is None
    assert m.apply(walk([a, h, b], gang=True)) is None
    # the bound table stays through bs_update_groups and goes with bs_update_nodes and bs_upload_groups
    assert m.apply({"op": "update_groups", "idx": np.array([0], np.uint32), "rows": snap.groups.take([0])}) is None
    assert m.bound is not None
    assert m.apply({"op": "upload_groups", "table": snap.groups}) is None and m.bound is None


def _fit_keys(pt):
    """Each pod's fit class key without the filter (engine.cu bs_upload_pods): (sel, tol, scalar keys requested with a
    non-zero amount, affinity class)."""
    nz = np.zeros(pt.n, np.uint64)
    for d in range(4, pt.lanes):
        nz |= ((((pt.req_present >> np.uint32(d)) & 1) == 1) & (pt.req[d] != 0)).astype(np.uint64) << np.uint64(d)
    aff = pt.aff_class if pt.aff_class is not None else np.full(pt.n, S.AFF_NONE, np.uint32)
    return list(zip(pt.sel_mask.tolist(), pt.tol_mask.tolist(), nz.tolist(), aff.tolist()))


def test_filter_rounds_follow_every_change():
    """Across the seeds, rounds with the filter on succeed right after a node table of another size, a node row
    update, a pod table refused for its lane count and a compaction of the fit class index; walks and preemption with
    PodDisruptionBudget bits succeed after row updates.  The compaction is certain once the (fit class, filter class)
    keys assigned since the last pod table outnumber max(4096, 4 x 2P), since the index only grows until it is
    compacted and a compaction keeps at most 2P classes (each pod's class and its class without the filter)."""
    reached, walks, pdb = set(), 0, 0
    for seed in SEEDS:
        ops, _, L = em.generate(seed)
        m = em.Model(L)
        pending, keys, n_prev, updated = set(), set(), None, False
        for op in ops:
            rc = m.apply(op)
            k = op["op"]
            if k == "upload_nodes" and rc is None:
                if n_prev is not None and op["table"].n != n_prev:
                    pending.add("resize")
                n_prev = op["table"].n
            elif k == "update_nodes" and rc is None and len(op["idx"]):
                pending.add("update_nodes")
                updated = True
            elif k == "update_groups" and rc is None:
                updated = True
            elif k == "upload_pods":
                if rc == em.E_INVAL:
                    pending.add("refused pods")
                elif rc is None:
                    keys = set()
            elif k == "evaluate" and rc is None and m.ipf_on:
                base = _fit_keys(m.pods)
                keys |= set(zip(base, m.ipf_pod[0].tolist()))
                if len(keys) > max(4096, 8 * m.pods.n):
                    pending.add("compaction")
                    keys = set()
                reached |= pending
                pending = set()
            elif k == "preempt_walk" and rc is None and updated and len(op["pods"]):
                walks += 1
            elif k == "preempt" and rc is None and updated and (m.bound.flags & S.BOUND_PDB_VIOLATING).any():
                pdb += 1
    assert reached == {"resize", "update_nodes", "refused pods", "compaction"}, reached
    assert walks >= 1 and pdb >= 1, (walks, pdb)


def test_expect_under_the_filter():
    """The round under the filter: filtered feasible counts never exceed the plain ones, each companion row sums to
    the nodes that fit the plain round and fail the filter, the Filter matrix and its codes are the same with the
    switch on and off, and the outputs the filter does not reach are the plain round's."""
    cfg = dict(score=True, fit_bitmap=True, filter=True, reasons=True, priority_k=8)
    for seed in (31, 32):
        m, snap, node, pods = _loaded(seed, P=120, N=200, G=20, L=[5, 9][seed % 2])
        assert m.apply({"op": "evaluate", "priority": True}) is None
        off = m.expect(cfg)
        assert not off["interpod_rows"].any()
        assert m.apply({"op": "ipf_switch", "on": True}) is None
        assert m.apply({"op": "evaluate", "priority": True}) is None
        on = m.expect(cfg)
        assert (on["feasible_count"] <= off["feasible_count"]).all()
        assert (on["feasible_count"] < off["feasible_count"]).any()
        N = snap.nodes.n
        fit = np.unpackbits(off["fit_rows"].view(np.uint8), axis=1, bitorder="little")[:, :N].astype(bool)
        v = fr.verdicts((node, pods), N)
        np.testing.assert_array_equal(on["interpod_rows"].sum(1), (fit & (v != fr.PASS)).sum(1))
        assert on["interpod_rows"].any()
        for key in ("filter_rows", "filter_code", "prefilter", "new_denied", "order", "rank", "reason_rows",
                    "max_group", "max_finished"):
            np.testing.assert_array_equal(on[key], off[key], err_msg=key)
        fit_on = np.unpackbits(on["fit_rows"].view(np.uint8), axis=1, bitorder="little")[:, :N].astype(bool)
        np.testing.assert_array_equal(fit_on, fit & (v == fr.PASS))
        assert (on["priority_nodes"] >= 0).sum(1).tolist() == np.minimum(8, on["feasible_count"]).tolist()


def _hp_half(snap, h, cols, n=None):
    return {"op": "hp", "half": h, "cols": cols, "n": (snap.nodes.n if h == "node" else snap.pods.n) if n is None else n}


def test_host_port_drop_rules_and_check_order():
    m, snap, node, pods = _loaded()
    N, P = snap.nodes.n, snap.pods.n
    (entries, used), want = hr.random_columns(snap, 4)
    assert want.any()
    ev = {"op": "evaluate", "priority": True}
    nz_node = {"op": "side", "name": "nz", "half": "node", "n": N, "cols": S.nonzero_requests(snap, 1)[0]}
    nz_pod = {"op": "side", "name": "nz", "half": "pod", "n": P, "cols": S.nonzero_requests(snap, 1)[1]}
    assert m.apply({"op": "hp_switch", "on": True}) is None
    assert m.apply(ev) == em.E_STATE                       # no halves
    assert m.apply(_hp_half(snap, "node", (entries, used))) is None
    assert m.apply(ev) == em.E_STATE                       # no pod half
    assert m.apply(_hp_half(snap, "pod", want)) is None
    assert m.apply(ev) is None and m.hp_round and not m.ipf_round
    # bs_update_nodes drops the node half, also a call that changes no row or fails
    for idx, rows in ((np.zeros(0, np.uint32), snap.nodes.take(np.zeros(0, np.int64))),
                      (np.array([N], np.uint32), snap.nodes.take([0])), (np.array([1], np.uint32), snap.nodes.take([1]))):
        m.apply({"op": "update_nodes", "idx": idx, "rows": rows})
        assert m.hp_node is None and m.hp_pod is not None
        assert m.apply(nz_node) is None
        assert m.apply(ev) == em.E_STATE
        assert m.apply(_hp_half(snap, "node", (entries, used))) is None
        assert m.apply(ev) is None
    # bs_upload_nodes drops it, also one that fails validation
    bad = snap.nodes.copy()
    bad.alloc[0, 0] = em.LIMIT + 1
    assert m.apply({"op": "upload_nodes", "table": bad}) == em.E_RANGE and m.hp_node is None
    assert m.apply(_hp_half(snap, "node", (entries, used))) == em.E_STATE   # without its table
    for op in ({"op": "upload_nodes", "table": snap.nodes}, {"op": "upload_affinity", "bits": snap.aff_bits}, nz_node,
               {"op": "ipf", "half": "node", "n": N, "cols": node}):
        assert m.apply(op) is None
    assert m.hp_node is None and m.apply(ev) == em.E_STATE
    # each failing node half leaves it dropped: a wrong length, more than 64 entries, a port outside 1..65535 (before
    # an entry listed twice), an entry listed twice (before a used bit past the entries), a used bit past the entries
    K = len(entries)
    twice = np.r_[entries[:-1], entries[:1]]
    zero_port = twice.copy()
    zero_port[0, 2] = 0
    past = used.copy()
    past[3] |= np.uint64(1) << np.uint64(K)
    many = np.array([(1, 0, 1000 + k) for k in range(65)], np.int64)
    for cols, n, rc in (((entries, used[:-1]), N - 1, em.E_INVAL), ((many, np.zeros(N, np.uint64)), N, em.E_INVAL),
                        ((zero_port, past), N, em.E_RANGE), ((twice, past), N, em.E_INVAL),
                        ((entries, past), N, em.E_INDEX)):
        assert m.apply(_hp_half(snap, "node", (entries, used))) is None
        assert m.apply(_hp_half(snap, "node", cols, n)) == rc and m.hp_node is None
    assert m.apply(_hp_half(snap, "node", (many[:64], np.zeros(N, np.uint64)))) is None   # 64 entries: every bit
    assert m.apply(ev) is None
    assert m.apply(_hp_half(snap, "node", (entries, used))) is None
    # bs_upload_pods drops the pod half and the placed side, also a call refused for its lane count (which keeps the
    # pod table and the node half)
    placed = S.node_interpod_walk(snap, 3)[2]
    assert m.apply({"op": "placed", "n": P, "cols": placed}) is None
    other = random_snapshot(5, P=7, N=1, G=1, L=6).pods
    assert m.apply({"op": "upload_pods", "table": other}) == em.E_INVAL
    assert m.pods is snap.pods and m.hp_pod is None and m.ipf_placed is None and m.hp_node is not None
    assert m.apply(nz_pod) is None
    assert m.apply(ev) == em.E_STATE
    assert m.apply(_hp_half(snap, "pod", want[:-1], P - 1)) == em.E_INVAL and m.hp_pod is None
    assert m.apply(_hp_half(snap, "pod", want)) is None
    assert m.apply(ev) is None
    # bs_evaluate: the priority sides, then the inter-pod filter, then the ports filter, then the affinity ids
    small = (entries[:1], used & np.uint64(1))     # the pods want entries past this dictionary
    assert m.apply(_hp_half(snap, "node", small)) is None
    assert m.apply(ev) == em.E_INDEX
    assert m.apply({"op": "weights", "w_spread": 1}) is None
    assert m.apply(ev) == em.E_STATE                       # the spread sides come first
    assert m.apply({"op": "weights", "w_spread": 0}) is None
    assert m.apply({"op": "ipf_switch", "on": True}) is None
    assert m.apply({"op": "ipf", "half": "pod", "n": P, "cols": (np.r_[pods[0][:-1], 0], pods[1])}) is None
    assert m.apply({"op": "ipf", "half": "node", "n": N + 1, "cols": node}) == em.E_INVAL
    assert m.apply(ev) == em.E_STATE                       # the inter-pod filter's half before the ports' dictionary
    assert m.apply({"op": "ipf", "half": "node", "n": N, "cols": node}) is None
    assert m.apply(ev) == em.E_INDEX
    assert m.apply({"op": "ipf_switch", "on": False}) is None
    assert m.apply({"op": "upload_affinity", "bits": None}) is None
    assert m.apply(_hp_half(snap, "pod", want[:-1], P - 1)) == em.E_INVAL
    assert m.apply(ev) == em.E_STATE                       # the ports filter before the affinity ids
    assert m.apply(_hp_half(snap, "pod", np.zeros(P, np.uint64))) is None
    assert m.apply(ev) == em.E_INDEX                       # now the affinity ids
    assert m.apply({"op": "upload_affinity", "bits": snap.aff_bits}) is None
    assert m.apply(ev) is None
    # preemption and the preemption walk are refused with the switch on, before the bound table is looked at
    for op in ({"op": "preempt", "pods": np.arange(5, dtype=np.uint32)},
               {"op": "preempt_walk", "pods": np.zeros(2, np.uint32), "gang": False}):
        assert m.apply(op) == em.E_INVAL
    assert m.apply({"op": "hp_switch", "on": False}) is None
    assert m.apply(ev) is None and not m.hp_round
    assert m.apply({"op": "preempt", "pods": np.arange(5, dtype=np.uint32)}) == em.E_STATE


def test_walk_refusals_under_the_filters():
    """bs_replay / bs_replay_priority with the filters: the inter-pod filter without the placed side first, then the
    priority weights, the tables, the non-zero columns, locality, the ports filter, the inter-pod filter, a placed
    term past the filter's dictionary; the placed side's own refusals; with the filter off it is not read."""
    m, snap, node, pods = _loaded()
    N, P = snap.nodes.n, snap.pods.n
    ff, pr = {"op": "replay", "priority": False}, {"op": "replay", "priority": True}
    placed = S.node_interpod_walk(snap, 3)[2]
    pcls, (off, term, own, match) = placed
    T = len(node[2])
    far = (pcls, (off, np.where(np.arange(len(term)) == 0, T, term).astype(np.uint32), own, match))
    pl = lambda cols, n=P: {"op": "placed", "n": n, "cols": cols}
    assert m.apply(ff) is None and m.apply(pr) is None
    assert m.apply({"op": "ipf_switch", "on": True}) is None
    assert m.apply({"op": "hp_switch", "on": True}) is None
    assert m.apply(ff) == em.E_INVAL                        # no placed side, before the ports filter's E_STATE
    assert m.apply({"op": "weights", "w_spread": 1}) is None
    assert m.apply(pr) == em.E_INVAL
    # the placed side's refusals: its table, its length, a class out of range, an own outside {0, 1}
    assert m.apply(pl(placed, P + 1)) == em.E_INVAL and m.ipf_placed is None
    assert m.apply(pl((np.full(P, len(off) - 1, np.uint32), placed[1]))) == em.E_INDEX
    bad_own = (pcls, (off, term, np.where(np.arange(len(own)) == 0, 2, own).astype(np.int32), match))
    assert len(own) and m.apply(pl(bad_own)) == em.E_RANGE and m.ipf_placed is None
    assert m.apply(pl(far)) is None                          # a term past the dictionary is checked by the walk
    assert m.apply(pr) == em.E_INVAL                         # bs_replay_priority's weights next
    assert m.apply({"op": "weights", "w_spread": 0}) is None
    assert m.apply(pr) == em.E_STATE and m.apply(ff) == em.E_STATE   # the ports filter's halves before the placed term
    (entries, used), want = hr.random_columns(snap, 4)
    assert m.apply(_hp_half(snap, "node", (entries[:1], used & np.uint64(1)))) is None
    assert m.apply(_hp_half(snap, "pod", want)) is None
    assert m.apply(ff) == em.E_INDEX                         # want bits past the dictionary
    assert m.apply({"op": "weights", "lw": (1, 0)}) is None
    assert m.apply(pr) == em.E_STATE                         # locality before the ports filter
    assert m.apply({"op": "weights", "lw": (0, 0)}) is None
    assert m.apply(_hp_half(snap, "node", (entries, used))) is None
    assert m.apply({"op": "ipf", "half": "pod", "n": P, "cols": (pods[0], (pods[1][0], np.full_like(pods[1][1], T),
                                                                          *pods[1][2:]))}) is None
    assert m.apply(ff) == em.E_INDEX                         # the pods' filter terms
    assert m.apply({"op": "ipf", "half": "pod", "n": P, "cols": pods}) is None
    assert m.apply(ff) == em.E_INDEX and m.apply(pr) == em.E_INDEX   # now the placed term
    assert m.apply({"op": "ipf_switch", "on": False}) is None
    assert m.apply(ff) is None and m.apply(pr) is None       # the placed side is not read
    assert m.apply({"op": "upload_pods", "table": snap.pods}) is None and m.ipf_placed is None
    assert m.apply({"op": "ipf_switch", "on": True}) is None
    assert m.apply(ff) == em.E_INVAL


def _conflicts(entries):
    """Each entry's conflict mask (engine.cu bs_upload_node_host_ports)."""
    ent = np.asarray(entries, np.int64).reshape(-1, 3)
    out = []
    for a in ent:
        same = (ent[:, 1] == a[1]) & (ent[:, 2] == a[2]) & ((ent[:, 0] == 0) | (a[0] == 0) | (ent[:, 0] == a[0]))
        out.append(sum(1 << int(b) for b in np.flatnonzero(same)))
    return out


def _fit_index_grows(seed):
    """(rounds that certainly compacted the fit class index with the ports filter on, ops, Model): a round is certain
    to compact once the (base class, filter class, conflict mask) keys assigned since the last pod table outnumber
    max(4096, 4 x 2P), as test_filter_rounds_follow_every_change reasons."""
    ops, _, L = em.generate(seed)
    m = em.Model(L)
    keys, hits = set(), []
    for i, op in enumerate(ops):
        rc = m.apply(op)
        if op["op"] == "upload_pods" and rc is None:
            keys = set()
        if op["op"] == "evaluate" and rc is None and (m.ipf_on or m.hp_on):
            ipf = m.ipf_pod[0].tolist() if m.ipf_on else [S.IPF_NONE] * m.pods.n
            conf = [0] * m.pods.n
            if m.hp_on:
                c = _conflicts(m.hp_node[0])
                conf = [functools.reduce(operator.or_, (c[b] for b in range(len(c)) if (int(w) >> b) & 1), 0)
                        for w in m.hp_pod]
            keys |= set(zip(_fit_keys(m.pods), ipf, conf))
            if len(keys) > max(4096, 8 * m.pods.n):
                hits.append(i)
                keys = set()
    return hits, ops, m


def test_r11_compacts_the_fit_index_under_the_ports_filter():
    seed = next(s for s in SEEDS if em.BURSTS[s % len(em.BURSTS)] == "r11")
    hits, ops, _ = _fit_index_grows(seed)
    assert hits, "R11 never outgrew the fit index"
    assert any(ops[i]["op"] == "evaluate" for i in hits)
    last_pods = max(i for i, op in enumerate(ops) if op["op"] == "upload_pods" and op["table"].n == 50)
    assert hits[0] < last_pods     # ... and then the small pod table


def test_r10_wants_again_after_a_refused_pod_table():
    """R10: a pod table refused for its lane count while the ports filter is on (after a round that gave the pods
    their conflict classes), then a want half other than the one before, then a successful round that changes what
    passes: the engine must build the classes from the base classes, not from the ones the filter gave them."""
    seed = next(s for s in SEEDS if em.BURSTS[s % len(em.BURSTS)] == "r10")
    ops, _, L = em.generate(seed)
    m = em.Model(L)
    found = False
    refused, want_before, want_after = None, None, None
    for op in ops:
        rc = m.apply(op)
        if op["op"] == "upload_pods":
            refused = m.hp_round and m.hp_on and rc == em.E_INVAL
            want_after = None
        elif op["op"] == "hp" and op["half"] == "pod" and rc is None:
            if refused and want_after is None:
                want_after = op["cols"]
            else:
                want_before = op["cols"]
        elif op["op"] == "evaluate" and rc is None and refused and want_after is not None and m.hp_on:
            found = found or not np.array_equal(want_after, want_before)
            refused = False
    assert found


def test_r12_walks_right_after_a_filter_half():
    """Across the seeds: successful filtered walks (first fit and priority) right after a filter half and before any
    round, under the inter-pod filter, the ports filter and both, and walks with the placed side refused."""
    reached = set()
    for seed in SEEDS:
        ops, _, L = em.generate(seed)
        m = em.Model(L)
        fresh = False
        for op in ops:
            rc = m.apply(op)
            if op["op"] in ("ipf", "hp") and rc is None:
                fresh = True
            elif op["op"] == "evaluate":
                fresh = False
            elif op["op"] == "replay" and rc is None and fresh and (m.ipf_on or m.hp_on):
                on = "both" if m.ipf_on and m.hp_on else ("ipf" if m.ipf_on else "hp")
                reached.add((on, "priority" if op["priority"] else "first_fit"))
    assert reached == {(on, k) for on in ("ipf", "hp", "both") for k in ("first_fit", "priority")}, reached


def test_walk_references_agree():
    """The model's walk references where two apply: interpod_walk_ref.replay with a filter without terms equals
    host_ports_ref.replay with the ports filter on, and the oracle's walk and locality_priority_ref.replay_locality
    with it off."""
    for seed, L in ((41, 5), (42, 6), (43, 9)):
        snap = random_snapshot(seed, P=90, N=120, G=14, L=L, aff=2)
        cols, placed = em.no_interpod_filter(snap.nodes.n, snap.pods.n)
        hp = hr.random_columns(snap, seed, node_bits=3, grouped=0.6)
        nz = S.nonzero_requests(snap, seed)
        for chooser in (None, nz):
            got = iwr.replay(snap, cols, placed, None, chooser, (1, 0, 1), None, None, (0, 0), hp)
            want = hr.replay(snap, hp, None, chooser, (1, 0, 1))
            for a, b in zip(got[:3], want[:3]):
                np.testing.assert_array_equal(a, b)
            np.testing.assert_array_equal(got[5], want[4])      # the live used masks
        assert (got[1] >= 0).any() and (hr.passes(*hp[0], hp[1]) == 0).any()
        got = iwr.replay(snap, cols, placed)
        want = oracle.replay(snap)
        for a, b in zip(got[:3], want[:3]):
            np.testing.assert_array_equal(a, b)
        loc = S.node_locality(snap, seed)
        ratio = (2, em.RATIO_ON[1], [1, 1, 0, 0] + [1] * (L - 4), 1)
        got = iwr.replay(snap, cols, placed, None, nz, (1, 0, 1), ratio, loc, em.LW)
        want = lpr.replay_locality(snap, nz[0], nz[1], loc, em.LW, ratio, None, (1, 0, 1))
        for a, b in zip(got[:3], want[:3]):
            np.testing.assert_array_equal(a, b)
