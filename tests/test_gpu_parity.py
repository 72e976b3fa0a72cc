"""GPU parity tests: the CUDA path (through the C ABI) against the CPU oracle, bit-exact."""
import numpy as np
import pytest

from parity import run_and_compare, assert_round_equal
from randsnap import random_snapshot

pytestmark = pytest.mark.gpu


def test_core_test_go_cases(pkg, oracle, snapshot_mod):
    # pkg/scheduler/core/core_test.go:82-112 through the engine: fit bits true,false,false
    snap, expected, left_exp = snapshot_mod.core_test_cases()
    res, orc = run_and_compare(pkg, oracle, snap)
    assert list(res.feasible_count) == [1, 0, 0]
    eng = pkg.Engine(snap.lanes)
    eng.upload_nodes(snap.nodes)
    left, pres = eng.node_left(0, 0, 1.0)
    eng.close()
    assert list(left[:, 0]) == [9000, 0, 0, 99, 9, 19] and pres[0] == 0x30


def test_readme_snapshot(pkg, oracle, snapshot_mod):
    snap = snapshot_mod.readme_scenario()
    res, _ = run_and_compare(pkg, oracle, snap)
    assert (res.feasible_count == 1).all()
    # first pods of both groups in one frozen round: group1 is max (nil rule), matched==0 ->
    # pct 1.0 check of each pod's own group: 7100 >= 5000 for both -> every pod passes
    assert (res.prefilter == 0).all()
    assert list(res.admit) == [snapshot_mod.ADMIT, snapshot_mod.ADMIT]


def test_readme_second_round_denies_group2(pkg, oracle, snapshot_mod):
    # after group1's first pod is permitted (matched=1, requested 1900m): Appendix C step 2
    S = snapshot_mod
    snap = S.readme_scenario()
    snap.groups.matched[0] = 1
    snap.groups.flags[:] = S.GROUP_HAS_POD | S.GROUP_HAS_MINRES
    snap.groups.min_res[0, :] = 1000
    snap.nodes.requested[0, 0] = 1900
    snap.nodes.pod_count[0] = 5
    res, _ = run_and_compare(pkg, oracle, snap)
    assert (res.prefilter[:5] == S.PF_PASS).all()          # max group passes (core.go:150-155)
    assert (res.prefilter[5:] == S.PF_NOT_ENOUGH).all()    # 5600-1900=3700 < 4000+1000
    assert list(res.new_denied) == [0, 1]
    assert res.admit[1] == S.UNSCHEDULABLE


@pytest.mark.parametrize("cfg,scale", [(2, 1.0), (3, 0.06), (4, 0.05), (5, 0.012)])
def test_baseline_configs(pkg, oracle, snapshot_mod, cfg, scale):
    snap = snapshot_mod.config(cfg, scale)
    run_and_compare(pkg, oracle, snap)


@pytest.mark.parametrize("cfg,scale", [(2, 0.5), (3, 0.04)])
def test_baseline_configs_case_a(pkg, oracle, snapshot_mod, cfg, scale):
    # no carried-in matched pods: every group is checked against its own need at pct 1.0
    snap = snapshot_mod.config(cfg, scale)
    snap.groups.matched[:] = 0
    res, orc = run_and_compare(pkg, oracle, snap)
    assert orc.max_group >= 0


@pytest.mark.parametrize("seed", range(24))
def test_random_snapshots(pkg, oracle, seed):
    case = ["mixed", "A", "B"][seed % 3]
    L = [4, 5, 6, 9, 16][seed % 5]
    snap = random_snapshot(seed, P=150 + 37 * seed, N=33 + 29 * seed, G=5 + 3 * seed, L=L, case=case,
                           value_scale="big" if seed % 7 == 3 else "normal")
    run_and_compare(pkg, oracle, snap)


def test_ragged_and_empty(pkg, oracle, snapshot_mod):
    S = snapshot_mod
    # no pods
    snap = random_snapshot(100, P=0, N=10, G=4, L=5)
    run_and_compare(pkg, oracle, snap)
    # no groups: every pod ungrouped or missing
    snap = random_snapshot(101, P=50, N=10, G=0, L=5)
    run_and_compare(pkg, oracle, snap)
    # single node, node count not a multiple of 32, > one tile
    for n in (1, 31, 32, 33, 511, 512, 513, 1100):
        snap = random_snapshot(200 + n, P=70, N=n, G=6, L=5)
        run_and_compare(pkg, oracle, snap, score=(n < 600))
    # empty snapshot list: every cluster check is false (core.go:604,631)
    for case in ("A", "B"):
        snap = random_snapshot(103, P=40, N=0, G=5, L=5, case=case)
        res, _ = run_and_compare(pkg, oracle, snap)
        assert (res.feasible_count == 0).all()
    # every node skipped: the cluster loop never compares (core.go:606-631)
    snap = random_snapshot(102, P=40, N=20, G=5, L=5, case="A")
    snap.nodes.flags[:] = S.NODE_UNSCHEDULABLE
    res, _ = run_and_compare(pkg, oracle, snap)
    assert (res.feasible_count == 0).all()


def test_uint32_wraparound_permit(pkg, oracle, snapshot_mod):
    # Status.Scheduled > MinMember: MinMember - Scheduled wraps (core.go:303, quirk Q6)
    S = snapshot_mod
    snap = S.readme_scenario()
    snap.groups.min_member[:] = [2, 5]
    snap.groups.scheduled[:] = [3, 0]
    res, orc = run_and_compare(pkg, oracle, snap)
    assert res.admit[0] == S.WAIT  # 5 pods < 2^32-1


def test_ref_panic_reported(pkg, snapshot_mod):
    S = snapshot_mod
    snap = S.readme_scenario()
    snap.groups.min_member[0] = 0
    snap.groups.scheduled[0] = 1
    eng = pkg.Engine(snap.lanes)
    eng.upload(snap)
    with pytest.raises(pkg.capi.BsError) as ei:
        eng.evaluate()
    assert ei.value.code == pkg.capi.BS_E_REF_PANIC
    eng.close()


@pytest.mark.parametrize("seed", range(6))
def test_node_left_and_cluster_check(pkg, oracle, seed):
    snap = random_snapshot(300 + seed, P=10, N=150 + 100 * seed, G=3, L=[5, 6, 9][seed % 3])
    nt = snap.nodes
    rng = np.random.default_rng(seed)
    eng = pkg.Engine(snap.lanes)
    eng.upload_nodes(nt)
    for sel, tol, pct in [(0, 0, 1.0), (1, 3, 0.7), (2, 0, 0.7), (5, 1, 1.0)]:
        left, pres = eng.node_left(sel, tol, pct)
        oleft, opres = oracle.node_left(nt, sel, tol, pct)
        np.testing.assert_array_equal(left, oleft)
        np.testing.assert_array_equal(pres, opres)
        total, tp = oracle.compute_cluster(nt, sel, tol)
        n_needs = 64
        need = np.zeros((snap.lanes, n_needs), np.int64)
        for d in range(snap.lanes):
            hi = max(2, int(abs(total[d])) * 2)
            need[d] = rng.integers(-hi // 4, hi, n_needs)
        need[:, :8] = 0
        need[3, :] = rng.integers(0, 50, n_needs)
        npres = rng.integers(0, 1 << snap.lanes, n_needs).astype(np.uint32) & ~np.uint32(0xF)
        ok = eng.cluster_check(sel, tol, pct, need, npres)
        exp = np.array([oracle.compare_cluster(nt, sel, tol, need[:, i], int(npres[i]), pct)
                        for i in range(n_needs)])
        np.testing.assert_array_equal(ok, exp)
    eng.close()


def test_mirrors_prefilter_permit_less(pkg, oracle, snapshot_mod):
    S = snapshot_mod
    snap = random_snapshot(77, P=120, N=40, G=12, L=5)
    snap.pods.flags[:10] |= S.POD_LISTER_MISS
    eng = pkg.Engine(snap.lanes)
    eng.upload(snap)
    eng.set_wait_time(0, None)
    res = eng.evaluate()
    orc = oracle.round(snap)
    capi = pkg.capi
    for p in range(snap.pods.n):
        code, reason, g = eng.prefilter(p)
        assert reason == orc.prefilter[p]
        assert code == (capi.CODE_SUCCESS if reason == 0 else capi.CODE_UNSCHEDULABLE)  # batchscheduler.go:104-107
        pr = eng.permit(p, 0)
        gid = snap.pods.gid[p]
        if gid == S.GID_NONE:
            assert pr["code"] == capi.CODE_SUCCESS and pr["wait_ns"] == 0
        elif gid < 0:
            assert pr["code"] == capi.CODE_UNSCHEDULABLE and pr["wait_ns"] == 60 * 10**9
        else:
            assert pr["code"] == capi.CODE_WAIT and pr["wait_ns"] == 10**9
            assert pr["ready"] == (orc.admit[gid] == S.ADMIT) and pr["start_signal"] == pr["ready"]
    rng = np.random.default_rng(5)
    for _ in range(3000):
        a, b = rng.integers(0, snap.pods.n, 2)
        assert eng.less(int(a), int(b)) == oracle.compare(snap.pods, snap.groups, int(a), int(b)), (a, b)
    assert eng.message(S.PF_NOT_ENOUGH) == "cluster resource not enough"
    assert eng.message(S.PF_NOT_FOUND, "default/g1") == "can not found pod group: default/g1"
    assert eng.message(S.PF_DENIED, "default/g1") == "pod with pgName: default/g1 last failed in 20s, deny"
    eng.close()


def test_value_range_rejected(pkg, oracle, snapshot_mod):
    snap = snapshot_mod.readme_scenario()
    snap.nodes.alloc[1, 0] = (1 << 56) + 1
    eng = pkg.Engine(snap.lanes)
    with pytest.raises(pkg.capi.BsError) as ei:
        eng.upload_nodes(snap.nodes)
    assert ei.value.code == pkg.capi.BS_E_RANGE
    eng.close()
    # a group / pod table that fails validation is dropped: the engine refuses to evaluate until a
    # valid one arrives (the DMA runs under the validation pass, so the old rows are gone)
    snap = snapshot_mod.readme_scenario()
    eng = pkg.Engine(snap.lanes)
    eng.upload(snap)
    eng.evaluate()
    bad = snap.groups.copy() if hasattr(snap.groups, "copy") else snap.copy().groups
    bad.min_res[0, 0] = -(1 << 57)
    with pytest.raises(pkg.capi.BsError) as ei:
        eng.upload_groups(bad)
    assert ei.value.code == pkg.capi.BS_E_RANGE
    with pytest.raises(pkg.capi.BsError) as ei:
        eng.evaluate()
    assert ei.value.code == pkg.capi.BS_E_STATE
    eng.upload_groups(snap.groups)
    assert (eng.evaluate().prefilter == 0).all()
    eng.close()
    # the same for a node table on an engine that already holds one: the old snapshot, its affinity table and its
    # bound-pod table go with the failed upload, and no round answers from them
    snap = random_snapshot(182, P=60, N=40, G=6, L=5, aff=2)
    eng = pkg.Engine(snap.lanes)
    eng.upload(snap)
    eng.upload_bound_pods(snapshot_mod.bound_pods(snap, 182))
    eng.evaluate()
    bad = snap.nodes.copy()
    bad.requested[0, 7] = (1 << 56) + 1
    calls = [lambda: eng.upload_nodes(bad), eng.evaluate, lambda: eng.update_nodes([0], snap.nodes.take([0])),
             lambda: eng.upload_affinity(snap.aff_bits), lambda: eng.preempt(np.arange(snap.pods.n))]
    for k, call in enumerate(calls):
        with pytest.raises(pkg.capi.BsError) as ei:
            call()
        assert ei.value.code == (pkg.capi.BS_E_RANGE if k == 0 else pkg.capi.BS_E_STATE), k
    eng.upload_nodes(snap.nodes)      # a valid table again: the affinity table has to follow it
    with pytest.raises(pkg.capi.BsError) as ei:
        eng.evaluate()
    assert ei.value.code == pkg.capi.BS_E_INDEX
    eng.upload_affinity(snap.aff_bits)
    res = eng.evaluate()
    eng.close()
    assert_round_equal(res, None, None, oracle.round(snap))


def test_reupload_and_reevaluate(pkg, oracle, snapshot_mod):
    # one engine, several rounds: state from a previous round must not leak
    eng = pkg.Engine(5, 0, fit_bitmap=True, score=True)
    for seed in (1, 2, 3):
        snap = random_snapshot(400 + seed, P=90 + 40 * seed, N=50 + 300 * seed, G=9 + seed, L=5)
        eng.upload(snap)
        for _ in range(2):
            res = eng.evaluate()
            orc = oracle.round(snap, want_bitmap=True, want_score=True)
            assert_round_equal(res, eng.fit_rows(), eng.score_rows(), orc)
        # numpy-style out=: the same arrays are refilled (and a stale shape is refused)
        res.prefilter[:] = 99
        again = eng.evaluate(out=res)
        assert again is res
        assert_round_equal(res, eng.fit_rows(), eng.score_rows(), orc)
        # back-to-back rounds without a sync in between, then one fetch: the three streams of a round
        # (fit, PreFilter chain, sort) must not run into the next round's
        for _ in range(3):
            eng.evaluate_async()
        eng.sync()
        assert_round_equal(eng.fetch(), eng.fit_rows(), eng.score_rows(), orc)
    with pytest.raises(ValueError):
        eng.upload(random_snapshot(77, P=33, N=20, G=4, L=5))
        eng.evaluate(out=res)
    eng.close()


@pytest.mark.parametrize("variant", ["all_narrow", "boundary", "cpu_wide", "many_scalars", "all_wide", "sentinel_mix"])
def test_lane_classification_variants(pkg, oracle, snapshot_mod, variant):
    """The fit kernel evaluates lanes whose values fit in 28 bits with 32-bit arithmetic and the
    rest in 64-bit; every wide/narrow split must give the same bits as the oracle."""
    S = snapshot_mod
    L = {"many_scalars": 13, "sentinel_mix": 9}.get(variant, 6)
    snap = random_snapshot(900 + len(variant), P=257, N=700, G=20, L=L)
    nt, pt = snap.nodes, snap.pods
    rng = np.random.default_rng(len(variant))
    N, P = nt.n, pt.n
    if variant in ("all_narrow", "boundary", "many_scalars", "sentinel_mix"):
        for d in range(L):
            hi = (1 << 26) if variant == "boundary" else 100000
            nt.alloc[d] = rng.integers(0, hi, N)
            nt.requested[d] = rng.integers(0, hi, N)
            pt.req[d] = rng.integers(0, 1 << 27 if variant == "boundary" else 50000, P)
            snap.groups.min_res[d] = rng.integers(0, 1000, snap.groups.n)
        if variant == "boundary":
            nt.alloc[0, 0] = 1 << 26           # still narrow
            nt.alloc[1, 0] = (1 << 26) + 1     # lane 1 becomes wide
            pt.req[2, 0] = 1 << 27             # still narrow
        nt.pod_count = rng.integers(0, 100, N).astype(np.int32)
        nt.requested[3] = 0
    if variant == "cpu_wide":
        nt.alloc[0] = rng.integers(1 << 30, 1 << 40, N)
        for d in (1, 2):
            nt.alloc[d] = rng.integers(0, 1 << 20, N)
            nt.requested[d] = rng.integers(0, 1 << 20, N)
            pt.req[d] = rng.integers(0, 1 << 19, P)
    if variant == "all_wide":
        for d in range(L):
            nt.alloc[d] = rng.integers(1 << 30, 1 << 45, N)
            pt.req[d] = rng.integers(0, 1 << 44, P)
    if variant == "sentinel_mix":
        # scalar lanes with absent keys on both sides: exercises the 32-bit sentinels
        nt.alloc_present = rng.integers(0, 1 << L, N).astype(np.uint32) & ~np.uint32(0xF)
        nt.req_present = rng.integers(0, 1 << L, N).astype(np.uint32) & ~np.uint32(0xF)
        pt.req_present = rng.integers(0, 1 << L, P).astype(np.uint32) & ~np.uint32(0xF)
        pt.req[4:] = rng.integers(0, 3, (L - 4, P))
        nt.flags[:] = 0
        nt.label_mask[:] = 0xF
        nt.taint_mask[:] = 0
    run_and_compare(pkg, oracle, snap)


@pytest.mark.parametrize("seed", range(8))
def test_filter_matrix(pkg, oracle, snapshot_mod, seed):
    """ScheduleOperation.Filter / computeResourceSatisfied (core.go:170-191, 514-564) per (pod,node)."""
    S = snapshot_mod
    snap = random_snapshot(700 + seed, P=130 + 60 * seed, N=40 + 150 * seed, G=8 + 2 * seed, L=[5, 6, 9][seed % 3],
                           case=["mixed", "B", "A"][seed % 3])
    if seed == 5:
        snap.groups.flags[:] |= S.GROUP_SCHEDULED      # no eligible group: maxPGStatus == nil (core.go:525)
    eng = pkg.Engine(snap.lanes, 0, fit_bitmap=False, score=False, filter=True)
    eng.upload(snap)
    res = eng.evaluate()
    rows = eng.filter_rows()
    orc = oracle.round(snap, want_bitmap=False, want_filter=True)
    np.testing.assert_array_equal(rows, orc.filter_bitmap)
    np.testing.assert_array_equal(res.filter_code, orc.filter_code)
    np.testing.assert_array_equal(res.prefilter, orc.prefilter)
    # per-call mirror on a sample of pairs
    rng = np.random.default_rng(seed)
    capi = pkg.capi
    for _ in range(40):
        p, n = int(rng.integers(0, snap.pods.n)), int(rng.integers(0, snap.nodes.n))
        code, reason, _ = eng.filter(p, n)
        bit = (orc.filter_bitmap[p, n >> 5] >> (n & 31)) & 1
        assert (reason == capi.FILTER_PASS) == bool(bit)
        assert code == (capi.CODE_SUCCESS if bit else capi.CODE_UNSCHEDULABLE)
        if not bit and orc.filter_code[p] == capi.FILTER_PASS:
            assert reason == (capi.FILTER_NO_SNAPSHOT if snap.nodes.flags[n] & S.NODE_NIL else capi.FILTER_NOT_ENOUGH)
    eng.close()


def test_out_of_memory_is_reported_not_fatal(pkg, snapshot_mod):
    # a score matrix that cannot fit (2M pods x 50k nodes x 8 B = 800 GB) must come back as BS_E_NOMEM,
    # and the engine must stay usable
    S = snapshot_mod
    big = S.config(5, 0.002)
    P = 2_000_000
    idx = np.arange(P) % big.pods.n
    snap = S.Snapshot(S.config(5, 1.0).nodes, big.pods.take(idx), big.groups)
    eng = pkg.Engine(snap.lanes, 0, fit_bitmap=False, score=True)
    eng.upload(snap)
    with pytest.raises(pkg.capi.BsError) as ei:
        eng.evaluate()
    assert ei.value.code == pkg.capi.BS_E_NOMEM
    small = random_snapshot(5, P=60, N=40, G=6, L=9)
    eng.upload(small)
    eng.evaluate()
    eng.close()


def test_find_max_tie_rule_on_gpu(pkg, oracle, snapshot_mod):
    """findMaxPG's order-dependent tie rule (core.go:725-735) through the parallel merge: many groups
    with equal progress, finished holders, Status.Scheduled==0 challengers, MinMember==0 chains."""
    S = snapshot_mod
    rng = np.random.default_rng(123)
    for trial in range(40):
        G = int(rng.integers(1, 3000))
        snap = random_snapshot(1000 + trial, P=64, N=20, G=G, L=4)
        gt = snap.groups
        gt.flags[:] = S.GROUP_HAS_POD | S.GROUP_HAS_MINRES
        gt.flags[rng.random(G) < 0.1] |= S.GROUP_SCHEDULED
        mode = trial % 4
        if mode == 0:      # everything at progress 0, mixed finished / unfinished holders
            gt.matched[:] = 0
            gt.min_member[:] = rng.choice([0, 1, 2, 5], G)
            gt.scheduled[:] = np.where(rng.random(G) < 0.5, gt.min_member, 0)
        elif mode == 1:    # equal non-zero progress everywhere
            gt.min_member[:] = 4
            gt.scheduled[:] = rng.choice([0, 0, 1], G)
            gt.matched[:] = 2 - gt.scheduled
        elif mode == 2:    # holder finished (scheduled > minMember wraps), challengers with Scheduled == 0
            gt.min_member[:] = rng.choice([1, 2, 3], G)
            gt.scheduled[:] = np.where(rng.random(G) < 0.3, gt.min_member, 0)
            gt.matched[:] = 0
        else:              # MinMember == 0 with Scheduled == 0 chains (0 >= 0 is "finished")
            gt.min_member[:] = rng.choice([0, 0, 3], G)
            gt.scheduled[:] = 0
            gt.matched[:] = 0
        gt.scheduled[(gt.min_member == 0) & (gt.scheduled != 0)] = 0   # avoid the divide-by-zero panic
        m, fin, panic = oracle.find_max_pg(snap.resolve_groups().groups)
        assert not panic
        eng = pkg.Engine(snap.lanes, 0, fit_bitmap=False, score=False)
        eng.upload(snap)
        res = eng.evaluate()
        eng.close()
        assert (res.max_group, res.max_finished) == (m, fin), (trial, mode, G)


def test_prefix_scratch_chunking(pkg, oracle, monkeypatch):
    """Case A with more representative classes than scratch slots: the class loop runs in chunks."""
    snap = random_snapshot(4242, P=400, N=300, G=60, L=6, case="A")
    rng = np.random.default_rng(1)
    snap.groups.rep_sel = rng.integers(0, 16, snap.groups.n).astype(np.uint64)    # many distinct classes
    snap.groups.rep_tol = rng.integers(0, 4, snap.groups.n).astype(np.uint64)
    snap.pods.sel_mask = rng.integers(0, 16, snap.pods.n).astype(np.uint64)
    snap.pods.tol_mask = rng.integers(0, 4, snap.pods.n).astype(np.uint64)
    monkeypatch.setenv("BS_PREFIX_BUDGET_BYTES", str(3 * 300 * (8 * 6 + 4)))       # 3 class slots
    run_and_compare(pkg, oracle, snap)


def test_concurrent_mirror_calls_are_safe(pkg, oracle, snapshot_mod):
    """Less / Permit / PreFilter are called from several goroutines in the reference
    (batchscheduler.go:165,214); one handle must serve concurrent callers."""
    import threading
    snap = random_snapshot(808, P=300, N=50, G=20, L=5)
    eng = pkg.Engine(snap.lanes, 0, fit_bitmap=True, score=False)
    eng.upload(snap)
    eng.evaluate()
    orc = oracle.round(snap)
    errors = []

    def worker(seed):
        rng = np.random.default_rng(seed)
        try:
            for _ in range(400):
                a, b = (int(x) for x in rng.integers(0, snap.pods.n, 2))
                assert eng.less(a, b) == oracle.compare(snap.pods, snap.groups, a, b)
                assert eng.prefilter(a)[1] == orc.prefilter[a]
                eng.permit(b, 0)
        except Exception as ex:  # noqa: BLE001
            errors.append(ex)
    ts = [threading.Thread(target=worker, args=(i,)) for i in range(8)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors[:1]
    eng.close()


def test_incremental_node_update(pkg, oracle, snapshot_mod):
    """bs_update_nodes: changing a few NodeInfos between cycles == re-uploading the whole snapshot."""
    S = snapshot_mod
    snap = random_snapshot(5150, P=220, N=900, G=14, L=5)
    other = random_snapshot(5151, P=10, N=900, G=2, L=5).nodes
    eng = pkg.Engine(snap.lanes, 0, fit_bitmap=True, score=True)
    eng.upload(snap)
    eng.evaluate()
    rng = np.random.default_rng(3)
    for round_ in range(3):
        idx = np.sort(rng.choice(snap.nodes.n, size=37, replace=False)).astype(np.uint32)
        rows = S.NodeTable(other.alloc[:, idx], other.requested[:, idx], other.pod_count[idx], other.alloc_present[idx],
                           other.req_present[idx], other.label_mask[idx], other.taint_mask[idx], other.flags[idx])
        if round_ == 2:   # a huge value flips a lane from narrow to wide
            rows.alloc[0, 0] = 1 << 40
        for f in ("alloc", "requested"):
            getattr(snap.nodes, f)[:, idx] = getattr(rows, f)
        for f in ("pod_count", "alloc_present", "req_present", "label_mask", "taint_mask", "flags"):
            getattr(snap.nodes, f)[idx] = getattr(rows, f)
        eng.update_nodes(idx, rows)
        res = eng.evaluate()
        orc = oracle.round(snap, want_bitmap=True, want_score=True)
        assert_round_equal(res, eng.fit_rows(), eng.score_rows(), orc)
    eng.close()


def test_incremental_group_update(pkg, oracle, snapshot_mod):
    """bs_update_groups: a few PodGroups change between cycles (matched, Scheduled, freeze flag, MinResources,
    representative pod, even creation time) == re-uploading the whole group table."""
    S = snapshot_mod
    snap = random_snapshot(6160, P=260, N=300, G=40, L=6)
    other = random_snapshot(6161, P=10, N=10, G=40, L=6, case="B").groups
    eng = pkg.Engine(snap.lanes, 0, fit_bitmap=True, score=True)
    eng.upload(snap)
    eng.evaluate()
    rng = np.random.default_rng(4)
    cols1 = ("min_member", "scheduled", "matched", "flags", "min_res_present", "rep_sel", "rep_tol", "creation_ns",
             "name_rank")
    for round_ in range(4):
        idx = np.sort(rng.choice(snap.groups.n, size=9, replace=False)).astype(np.uint32)
        rows = S.GroupTable(other.min_member[idx], other.scheduled[idx], other.matched[idx], other.flags[idx],
                            other.min_res[:, idx], other.min_res_present[idx], other.rep_sel[idx], other.rep_tol[idx],
                            other.creation_ns[idx], snap.groups.name_rank[idx])
        if round_ == 1:   # a representative class no pod of the round has
            rows.rep_sel[0] = np.uint64(0xF0F0)
            rows.flags[0] |= S.GROUP_HAS_POD
        if round_ == 2:   # a creation time with new high bits: more sort digits vary
            rows.creation_ns[1] = np.int64(1) << 61
        if round_ == 3:   # the walk continues from here as well
            rows.matched[:] = 0
        snap.groups.min_res[:, idx] = rows.min_res
        for f in cols1:
            getattr(snap.groups, f)[idx] = getattr(rows, f)
        eng.update_groups(idx, rows)
        res = eng.evaluate()
        orc = oracle.round(snap, want_bitmap=True, want_score=True)
        assert_round_equal(res, eng.fit_rows(), eng.score_rows(), orc)
        walk = eng.replay(res.order)
        pf, node, ready, _ = oracle.replay(snap, res.order)
        assert np.array_equal(walk["prefilter"], pf) and np.array_equal(walk["node"], node) and np.array_equal(walk["ready"], ready)
    with pytest.raises(Exception):
        eng.update_groups(np.array([snap.groups.n], np.uint32), S.GroupTable(*(getattr(rows, f)[..., :1] for f in (
            "min_member", "scheduled", "matched", "flags", "min_res", "min_res_present", "rep_sel", "rep_tol",
            "creation_ns", "name_rank"))))
    eng.close()


@pytest.mark.parametrize("seed", range(4))
def test_extreme_values(pkg, oracle, snapshot_mod, seed):
    """Corners of the value domain: magnitudes at +-2^56, negative capacities / requests, int64-extreme
    timestamps and creation times, uint32-extreme name ranks and counters, out-of-range group ids."""
    S = snapshot_mod
    rng = np.random.default_rng(900 + seed)
    snap = random_snapshot(9000 + seed, P=180, N=130, G=16, L=[5, 6, 9, 12][seed])
    nt, pt, gt = snap.nodes, snap.pods, snap.groups
    LIM = 1 << 56
    for d in range(snap.lanes):
        pick = rng.random(nt.n) < 0.3
        nt.alloc[d] = np.where(pick, rng.choice([LIM, LIM - 1, -LIM, 0, 1, -1, (1 << 26), (1 << 26) + 1], nt.n), nt.alloc[d])
        pick = rng.random(nt.n) < 0.3
        nt.requested[d] = np.where(pick, rng.choice([LIM, -LIM, 0, 1, -5, 1 << 55], nt.n), nt.requested[d])
        pick = rng.random(pt.n) < 0.3
        pt.req[d] = np.where(pick, rng.choice([LIM, -LIM, 0, -1, 1, (1 << 27), (1 << 27) + 1, 1 << 40], pt.n), pt.req[d])
        pick = rng.random(gt.n) < 0.3
        gt.min_res[d] = np.where(pick, rng.choice([LIM, -LIM, 0, 7, -7], gt.n), gt.min_res[d])
    nt.pod_count = rng.choice([0, 1, 2**31 - 1, -5, 100], nt.n).astype(np.int32)
    I64 = np.iinfo(np.int64)
    pt.ts_ns = rng.choice([I64.min, I64.max, 0, -1, 1, 10**18], pt.n)
    gt.creation_ns = rng.choice([I64.min, I64.max - 1, 0, -1, 1], gt.n)
    gt.name_rank = rng.choice([0, 1, 2**32 - 1, 2**31], gt.n).astype(np.uint32)
    gt.min_member = rng.choice([1, 2, 2**32 - 1, 2**31, 7], gt.n).astype(np.uint32)
    gt.scheduled = rng.choice([0, 1, 2**32 - 1, 7], gt.n).astype(np.uint32)
    gt.matched = rng.choice([0, 1, 2**32 - 1, 5000000], gt.n).astype(np.uint32)
    pt.gid = np.where(rng.random(pt.n) < 0.1, gt.n + 5, pt.gid).astype(np.int32)
    pt.priority = rng.choice([-2**31, 2**31 - 1, 0, -1, 1], pt.n).astype(np.int32)
    run_and_compare(pkg, oracle, snap)


@pytest.mark.parametrize("case", ["A", "B"])
def test_more_than_65535_classes(pkg, oracle, snapshot_mod, case):
    """Every pod its own selector/toleration class: class tables beyond one grid dimension
    (gridDim.y <= 65535) and beyond one prefix-scratch chunk."""
    rng = np.random.default_rng(77)
    snap = random_snapshot(6500, P=70000, N=64, G=300, L=5, case=case)
    snap.pods.sel_mask = rng.integers(0, 1 << 62, snap.pods.n).astype(np.uint64) & np.uint64(0xFFFFFFFFFFFFFFF0)
    snap.pods.sel_mask |= rng.integers(0, 16, snap.pods.n).astype(np.uint64)
    snap.pods.sel_mask[::7] = 0                      # some pods still fit somewhere
    snap.pods.tol_mask = rng.integers(0, 1 << 40, snap.pods.n).astype(np.uint64)
    snap.groups.flags &= ~np.uint8(snapshot_mod.GROUP_HAS_POD)   # representatives come from the pods
    run_and_compare(pkg, oracle, snap, score=False)


@pytest.mark.parametrize("seed", range(8))
def test_affinity_class_table(pkg, oracle, seed):
    """checkFit beyond the bit masks (core.go:741-759 -> PodMatchNodeSelector with required nodeAffinity
    terms): pods and group representatives carry an affinity class, the (class, node) verdicts come from the
    host as a bit table (bs_upload_affinity).  Every output of the round, bit-exact."""
    L = [4, 5, 6, 9][seed % 4]
    snap = random_snapshot(100 + seed, P=300 + 41 * seed, N=40 + 67 * seed, G=12 + 5 * seed, L=L,
                           case=["mixed", "A", "B"][seed % 3], aff=1 + seed % 5)
    run_and_compare(pkg, oracle, snap)


def test_affinity_semantics(pkg, oracle):
    """An all-ones row is no constraint; an all-zero row fits nowhere; a class id outside the table is an error."""
    S = pkg.snapshot
    base = random_snapshot(7, P=120, N=70, G=10, L=5)
    W = (base.nodes.n + 31) // 32
    ones = np.full((1, W), 0xFFFFFFFF, np.uint32)
    a = base.copy()
    a.aff_bits = ones
    a.pods.aff_class = np.zeros(a.pods.n, np.uint32)
    a.groups.rep_aff = np.zeros(a.groups.n, np.uint32)
    ra, _ = run_and_compare(pkg, oracle, a)
    rb, _ = run_and_compare(pkg, oracle, base)
    np.testing.assert_array_equal(ra.feasible_count, rb.feasible_count)
    np.testing.assert_array_equal(ra.prefilter, rb.prefilter)
    z = base.copy()
    z.aff_bits = np.zeros((2, W), np.uint32)
    z.aff_bits[1] = 0xFFFFFFFF
    z.pods.aff_class = np.zeros(z.pods.n, np.uint32)
    rz, _ = run_and_compare(pkg, oracle, z)
    assert rz.feasible_count.sum() == 0
    eng = pkg.Engine(base.lanes, 0)
    try:
        bad = base.copy()
        bad.pods.aff_class = np.full(bad.pods.n, 3, np.uint32)    # no table uploaded
        eng.upload(bad)
        with pytest.raises(pkg.capi.BsError) as ei:
            eng.evaluate()
        assert ei.value.code == pkg.capi.BS_E_INDEX
        bad.aff_bits = np.zeros((4, W), np.uint32)
        eng.upload(bad)
        eng.evaluate()
        eng.upload_nodes(bad.nodes)                               # a new node snapshot drops the table
        with pytest.raises(pkg.capi.BsError):
            eng.evaluate()
    finally:
        eng.close()


def test_stale_affinity_classes_do_not_count(pkg, oracle):
    """The engine's class indices outlive pod tables, so classes of an earlier table keep affinity ids that the table
    of now need not have.  A pod table without affinity classes, after a node upload that dropped the affinity table,
    evaluates and walks as on a fresh engine."""
    eng = pkg.Engine(5, 0)
    try:
        eng.upload(random_snapshot(41, P=90, N=60, G=8, L=5, aff=3))
        eng.evaluate()
        plain = random_snapshot(42, P=70, N=60, G=8, L=5)
        eng.upload(plain)
        res = eng.evaluate()
        walk = eng.replay(res.order)
    finally:
        eng.close()
    assert_round_equal(res, None, None, oracle.round(plain))
    pf, node, ready, _ = oracle.replay(plain, res.order)
    assert np.array_equal(walk["prefilter"], pf) and np.array_equal(walk["node"], node)
    assert np.array_equal(walk["ready"], ready)


def test_view_results_match_copies(pkg, oracle, snapshot_mod):
    """bs_evaluate_view / bs_fetch_view: the zero-copy decision vectors (pointers into the engine's pinned arena)
    hold exactly what bs_evaluate copies out, round after round, also after the tables change shape."""
    fields = ("prefilter", "feasible_count", "best_node", "best_score", "admit", "admit_bitmap", "new_denied", "order", "rank")
    eng = pkg.Engine(5, 0, fit_bitmap=True, score=True)
    for seed, (P, N, G) in enumerate([(300, 700, 25), (300, 700, 25), (90, 130, 7)]):
        snap = random_snapshot(8800 + seed, P=P, N=N, G=G, L=5)
        eng.upload(snap)
        v = eng.evaluate(view=True)
        orc = oracle.round(snap, want_bitmap=True, want_score=True)
        assert_round_equal(v, eng.fit_rows(), eng.score_rows(), orc)
        assert not v.prefilter.flags.writeable
        c = eng.fetch()            # the copying call answers from the same round
        v2 = eng.fetch(view=True)
        for f in fields:
            assert np.array_equal(getattr(v, f), getattr(c, f)), f
            assert np.array_equal(getattr(v2, f), getattr(c, f)), f
        assert (v.max_group, v.max_finished) == (c.max_group, c.max_finished)
    eng.close()
