"""CPU: the host model of a long-lived engine (tests/engine_model.py) and its op generator, without a device: row
updates through the model equal the tables built directly, the generator is deterministic and reaches every scripted
regime across the seeds the GPU test runs, and the model's expected outputs come from the restatements on a short
sequence (which keeps the reference side honest and bounds its cost)."""
import numpy as np

import engine_model as em
from randsnap import S, random_snapshot

SEEDS = range(8)


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
    assert seen == {"R1", "R2", "R3", "R4", "R5", "R6"}


def test_sequences_reach_the_edges():
    """Across the seeds: N, P and G of 0, node counts on both sides of the 512-node tile, the class indices past
    4096, every side refused once (wrong length), every error the model predicts, and a round after each."""
    codes, sizes, P_max = set(), set(), 0
    for seed in SEEDS:
        ops, _, L = em.generate(seed)
        m = em.Model(L)
        for op in ops:
            codes.add(m.apply(op))
            if op["op"] == "upload_nodes":
                sizes.add(op["table"].n)
            if op["op"] == "upload_pods":
                sizes.add(("P", op["table"].n))
                P_max = max(P_max, op["table"].n)
            if op["op"] == "upload_groups":
                sizes.add(("G", op["table"].n))
    assert {None, em.E_STATE, em.E_RANGE, em.E_INDEX, em.E_INVAL} <= codes
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
