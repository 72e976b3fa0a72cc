"""The cluster check where only the full prefix scan decides, through the engine: bs_cluster_check
(warp_cluster_check), case A rounds (group_check_kernel), case B rounds (prefilter_kernel's cooperative scan) and
bs_replay's block scan, on the designed tables of scan_cases.py, against the plain reference walk and the oracle."""
import numpy as np
import pytest

import scan_cases as sc
from parity import run_and_compare

pytestmark = pytest.mark.gpu

S = sc.S
TABLES = {t.name: t for t in sc.tables()}
NO_FIT = 1 << 40          # a pod selector no node carries: no pod is ever assumed, the node state stays as designed


def replay_both(pkg, oracle, snap, queue=None):
    eng = pkg.Engine(snap.lanes)
    eng.upload(snap)
    got = eng.replay(queue)
    eng.close()
    pf, node, ready, after = oracle.replay(snap, queue)
    np.testing.assert_array_equal(got["prefilter"], pf)
    np.testing.assert_array_equal(got["node"], node)
    np.testing.assert_array_equal(got["ready"], ready)
    np.testing.assert_array_equal(got["node_requested"], after.nodes.requested)
    np.testing.assert_array_equal(got["node_pod_count"], after.nodes.pod_count)
    np.testing.assert_array_equal(got["node_req_present"], after.nodes.req_present)
    np.testing.assert_array_equal(got["group_matched"], after.groups.matched)
    np.testing.assert_array_equal(got["group_flags"], after.groups.flags)
    np.testing.assert_array_equal(got["group_min_res"], after.groups.min_res)
    np.testing.assert_array_equal(got["group_min_res_present"], after.groups.min_res_present)
    np.testing.assert_array_equal(got["group_rep_sel"], after.groups.rep_sel)
    np.testing.assert_array_equal(got["group_rep_tol"], after.groups.rep_tol)
    return got


# ---------------------------------------------------------------------------------------------------------------
# a. bs_cluster_check

@pytest.mark.parametrize("name", sorted(TABLES) + ["one_node"])
def test_cluster_check(pkg, name):
    t = TABLES[name] if name in TABLES else sc.one_node_table()
    eng = pkg.Engine(t.lanes)
    eng.upload_nodes(t.nodes)
    try:
        for k, ((sel, tol), pct) in enumerate([(c, p) for c in sc.CLASSES for p in (1.0, 0.7)]):
            need, npres = sc.random_needs(t, sel, tol, pct, 250, seed=100 + k)
            if (sel, tol) == (sc.SEL, sc.TOL) and t.needs:
                # with alloc 0 the designed terms are the same at both percents
                dn, dp = sc.need_arrays(t.needs, t.lanes)
                need, npres = np.concatenate([dn, need], axis=1), np.concatenate([dp, npres])
            exp = sc.reference_answers(t, sel, tol, pct, need, npres)
            got = eng.cluster_check(sel, tol, pct, need, npres)
            bad = np.flatnonzero(got != exp)
            assert not len(bad), (name, (sel, tol), pct, [(need[:, j].tolist(), hex(npres[j]), exp[j]) for j in bad[:3]])
    finally:
        eng.close()


def fits_table_limits(need):
    """A need a group's MinResources or a pod's request can carry: the engine refuses table values beyond
    +-2^56 (BS_E_RANGE).  The base need of case B adds a few units."""
    return all(abs(int(x)) < (1 << 56) - 1000 for x in need)


# ---------------------------------------------------------------------------------------------------------------
# b. case A: every group against its own need at percent 1.0

def case_a_snapshot(t, n_random=120, seed=0):
    """One group (MinMember 1, Scheduled 0, matched 0) and one pod per need: the group's need is its MinResources.
    A pods-lane need of 0 would become MinMember + 1 (core.go:789-791), so the expected verdict uses that."""
    L = t.lanes
    rng = np.random.default_rng(seed)
    rows = [(n, p, sc.CLASSES[0]) for n, p, _, _ in t.needs]
    for k, cls in enumerate(sc.CLASSES):
        need, npres = sc.random_needs(t, cls[0], cls[1], 1.0, n_random // len(sc.CLASSES), seed=seed + k)
        rows += [(need[:, j].tolist(), int(npres[j]), cls) for j in range(need.shape[1])]
    rows = [r for r in rows if fits_table_limits(r[0])]
    order = rng.permutation(len(rows))
    rows = [rows[i] for i in order]
    G = len(rows)
    gt = S.GroupTable.empty(G, L)
    gt.min_member[:] = 1
    gt.flags[:] = S.GROUP_HAS_POD | S.GROUP_HAS_MINRES
    gt.creation_ns[:] = 1_600_000_000 * 10**9
    gt.name_rank[:] = np.arange(G)
    exp = np.zeros(G, bool)
    for g, (need, npres, (sel, tol)) in enumerate(rows):
        gt.min_res[:, g] = need
        gt.min_res_present[g] = npres
        gt.rep_sel[g], gt.rep_tol[g] = sel, tol
        eff = list(need)
        if eff[3] == 0:
            eff[3] = 2
        pre, keys, vis = sc.ref_prefixes(t, sel, tol, 1.0)
        exp[g] = sc.first_hit(pre, keys, vis, eff, npres) >= 0
    pt = S.PodTable.empty(G, L)
    pt.gid = np.arange(G, dtype=np.int32)
    pt.sel_mask[:] = NO_FIT
    pt.ts_ns = 1_700_000_000 * 10**9 + np.arange(G) * 1000
    snap = S.Snapshot(t.nodes, pt, gt, f"{t.name}_caseA")
    return snap, exp


@pytest.mark.parametrize("name", ["big", "edges", "scalar_keys", "leading_skip"])
def test_case_a_round(pkg, oracle, name):
    t = TABLES[name]
    snap, exp = case_a_snapshot(t)
    res, orc = run_and_compare(pkg, oracle, snap)
    assert res.max_group >= 0 and snap.groups.matched[res.max_group] == 0
    np.testing.assert_array_equal(res.prefilter, np.where(exp, S.PF_PASS, S.PF_NOT_ENOUGH))
    np.testing.assert_array_equal(res.new_denied, (~exp).astype(np.uint8))
    assert exp.any() and not exp.all()


def test_case_a_round_in_several_prefix_passes(pkg, oracle, monkeypatch):
    # room for 2 class slots: the 4 representative classes go through the prefix scan in passes
    t = TABLES["big"]
    snap, exp = case_a_snapshot(t, seed=3)
    monkeypatch.setenv("BS_PREFIX_BUDGET_BYTES", str(5 * t.nodes.n * (8 * t.lanes + 4) // 2))
    res, _ = run_and_compare(pkg, oracle, snap)
    np.testing.assert_array_equal(res.prefilter, np.where(exp, S.PF_PASS, S.PF_NOT_ENOUGH))


# ---------------------------------------------------------------------------------------------------------------
# c. case B: one max group with matched != 0, every other pod against its need plus the pod's request at 0.7

BASE_MIN_RES = [10, 20, 30, 1]      # max group 0: MinMember 4, matched 2 -> base need = 2 x MinResources


def case_b_snapshot(t, P=557, seed=0):
    """Pods in warps that mix decided and undecided needs: warp 0 undecided at lane 0 only, warp 1 at lane 31 only,
    warp 2 at four lanes, warp 3 entirely, then a random mix; P is not a multiple of 32 and spans three CTAs."""
    L = t.lanes
    rng = np.random.default_rng(seed)
    pre, keys, vis = sc.ref_prefixes(t, sc.SEL, sc.TOL, 0.7)
    st = sc.stats(pre, keys, vis)
    rows = [(n, p) for n, p, _, _ in t.needs]
    need, npres = sc.random_needs(t, sc.SEL, sc.TOL, 0.7, 300, seed=seed)
    rows += [(need[:, j].tolist(), int(npres[j])) for j in range(need.shape[1])]
    for d in range(L):                     # a few that the bounds reject
        row = [int(x) for x in pre[:, st.last_visited]]
        row[d] = st.maxv[d] + 1 if st.maxv[d] is not None else 1
        rows.append((row, sc.scalar_mask(L)))
    undecided, decided = [], []
    for row in rows:
        if fits_table_limits(row[0]):
            (undecided if sc.classify(pre, keys, vis, st, *row).startswith("step3") else decided).append(row)
    assert len(undecided) >= 4 and decided

    def pick(pool):
        return pool[int(rng.integers(len(pool)))]
    u_iter = iter(undecided * 40)
    lanes = [[0], [31], [3, 7, 8, 20], list(range(32))]
    rows = []
    for w in lanes:
        rows += [next(u_iter) if lane in w else pick(decided) for lane in range(32)]
    while len(rows) < P - 1:
        rows.append(next(u_iter) if rng.random() < 0.3 else pick(decided))
    G = P
    gt = S.GroupTable.empty(G, L)
    gt.min_member[:] = 1
    gt.creation_ns[:] = 1_600_000_000 * 10**9
    gt.name_rank[:] = np.arange(G)
    gt.min_member[0], gt.matched[0] = 4, 2
    gt.flags[0] = S.GROUP_HAS_POD | S.GROUP_HAS_MINRES
    gt.min_res[:4, 0] = BASE_MIN_RES
    gt.rep_sel[0], gt.rep_tol[0] = sc.SEL, sc.TOL
    base = [2 * x for x in BASE_MIN_RES]
    pt = S.PodTable.empty(P, L)
    pt.gid = np.arange(1, P + 1, dtype=np.int32)
    pt.gid[P - 1] = 0                       # the max group's own pod passes
    pt.sel_mask[:] = NO_FIT
    pt.ts_ns = 1_700_000_000 * 10**9 + np.arange(P) * 1000
    exp = np.ones(P, bool)
    for p, (n, npres) in enumerate(rows):
        pt.req[:4, p] = [n[d] - base[d] for d in range(4)]
        for d in range(4, L):
            if (npres >> d) & 1:
                pt.req[d, p] = n[d]
        pt.req_present[p] = npres
        exp[p] = sc.first_hit(pre, keys, vis, n, npres) >= 0
    snap = S.Snapshot(t.nodes, pt, gt, f"{t.name}_caseB")
    return snap, exp


@pytest.mark.parametrize("name", ["big", "leading_skip", "real_alloc", "edges"])
def test_case_b_round(pkg, oracle, name):
    t = TABLES[name]
    snap, exp = case_b_snapshot(t)
    m, _, panic = oracle.find_max_pg(snap.groups)
    assert m == 0 and not panic
    res, orc = run_and_compare(pkg, oracle, snap)
    assert res.max_group == 0 and orc.max_group == 0
    np.testing.assert_array_equal(res.prefilter, np.where(exp, S.PF_PASS, S.PF_NOT_ENOUGH))
    denied = np.zeros(snap.groups.n, np.uint8)
    denied[snap.pods.gid[~exp]] = 1
    np.testing.assert_array_equal(res.new_denied, denied)
    assert exp[:-1].any() and not exp.all()


# ---------------------------------------------------------------------------------------------------------------
# d. bs_replay: the block scan, its cached block summaries and its skip rule

@pytest.mark.parametrize("name,case", [("big", "A"), ("big", "B"), ("leading_skip", "B"), ("big_bump", "B"),
                                       ("big_bump", "A")])
def test_replay(pkg, oracle, name, case):
    """No pod fits a node, so the node state stays as designed for the whole walk, and each pod's group is its own:
    every queue position's verdict is the reference's verdict of its need.  In `big` each target is the maximum of
    its replay block on every lane >= 2, so carry + block maximum equals the need there exactly; `big_bump`'s sums
    pass 2^62, so the walk runs without the block cache."""
    t = TABLES[name]
    assert t.nodes.n >= 3 * 1024
    snap, exp = (case_a_snapshot if case == "A" else case_b_snapshot)(t)
    eng = pkg.Engine(snap.lanes)
    eng.upload(snap)
    order = eng.evaluate().order.copy()
    eng.close()
    got = replay_both(pkg, oracle, snap, order)
    np.testing.assert_array_equal(got["prefilter"], np.where(exp[order], S.PF_PASS, S.PF_NOT_ENOUGH))
