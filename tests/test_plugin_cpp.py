"""The C++ host mirror (batch-scheduler_b200/csrc/plugin.{hpp,cpp}): resource.Quantity parsing and the
snapshot packer on CPU; the README scenario pod-by-pod through BatchSchedulingPlugin on the GPU."""
import json
import subprocess

import numpy as np
import pytest

import native


@pytest.fixture(scope="module")
def plugin_bin():
    return native.cpp_program("plugin_test")


def _run(binary, *args):
    return json.loads(subprocess.check_output([binary, *args], text=True))


def test_quantity_parsing(plugin_bin):
    # (Value, MilliValue) as k8s resource.Quantity computes them (both round up)
    cases = {"1": (1, 1000), "900m": (1, 900), "140Mi": (140 << 20, (140 << 20) * 1000), "1.5": (2, 1500),
             "100": (100, 100000), "0": (0, 0), "1e3": (1000, 1000000), "2Gi": (2 << 30, (2 << 30) * 1000),
             "1k": (1000, 1000000), "0.5Gi": (1 << 29, (1 << 29) * 1000), "250u": (1, 1), "12E-1": None,
             "5G": (5 * 10**9, 5 * 10**12), "1Ki": (1024, 1024000), "-1": (-1, -1000), "1500m": (2, 1500)}
    out = _run(plugin_bin, "quantity", *cases)
    for s, exp in cases.items():
        ok, v, m = out[s]
        if exp is None:
            continue
        assert ok == 1 and (v, m) == exp, (s, out[s])
    bad = _run(plugin_bin, "quantity", "abc", "1Zi", "")
    assert all(v[0] == 0 for v in bad.values())


def test_packer_core_test_go(plugin_bin, snapshot_mod):
    # the objects of core_test.go:28-80 packed by the C++ packer == the hand-built tables
    snap, _, _ = snapshot_mod.core_test_cases()
    out = _run(plugin_bin, "pack_core_test")
    assert out["lanes"] == 6
    assert out["scalars"] == ["alpha.kubernetes.io/nvidia-gpu", "tencent.cr/tencentip"]
    assert out["alloc"] == snap.nodes.alloc.reshape(-1).tolist()
    assert out["requested"] == snap.nodes.requested.reshape(-1).tolist()
    assert out["pod_count"] == snap.nodes.pod_count.tolist()
    assert out["alloc_present"] == snap.nodes.alloc_present.tolist()
    assert out["req_present"] == snap.nodes.req_present.tolist()
    assert out["req"] == snap.pods.req.reshape(-1).tolist()
    assert out["pod_req_present"] == snap.pods.req_present.tolist()
    assert out["gid"] == [-1, -1, -1]


def test_packer_semantics(plugin_bin, snapshot_mod):
    """Hand-built objects through the C++ packer: every encoding the engine's tables rely on."""
    S = snapshot_mod
    o = _run(plugin_bin, "pack_semantics")
    N, P, G, L = 5, 7, 4, 6
    assert o["lanes"] == L and o["scalars"] == ["nvidia.com/gpu", "hugepages-2Mi"]   # first-seen order, IsScalarResourceName
    alloc = np.array(o["alloc"]).reshape(L, N)
    requested = np.array(o["requested"]).reshape(L, N)
    assert alloc[:, 0].tolist() == [4000, 8 << 30, 0, 110, 2, 1 << 30] and alloc[0].tolist() == [4000, 8000, 0, 0, 1000]
    assert requested[:, 0].tolist() == [500, 0, 0, 0, 1, 0] and o["pod_count"] == [3, 0, 0, 0, 0]
    assert o["alloc_present"] == [0x30, 0, 0, 0, 0] and o["req_present"] == [0x10, 0, 0, 0, 0]
    # nodeSelector pairs -> label bits; only NoSchedule / NoExecute taints get a bit (PodToleratesNodeTaints)
    assert o["label_mask"] == [1, 0, 0, 0, 1] and o["taint_mask"] == [1, 2, 0, 0, 0]
    assert o["node_flags"] == [0, S.NODE_UNSCHEDULABLE, S.NODE_NO_NODE, S.NODE_NIL, S.NODE_TAINTS_ERR]
    req = np.array(o["req"]).reshape(L, P)
    assert req[:, 0].tolist() == [1000, 1 << 30, 0, 0, 0, 0]      # Limits win over Requests when non-nil (Q10)
    assert req[:, 1].tolist() == [500, 0, 0, 0, 2, 0]             # two containers summed, Requests (Limits nil)
    assert req[:, 3].tolist() == [0] * L                          # Limits non-nil but empty: demand 0
    assert o["pod_req_present"] == [0, 0x10, 0, 0, 0, 0, 0]
    assert o["gid"] == [0, 0, S.GID_MISSING, S.GID_NONE, 1, 1, 0]
    assert o["sel_mask"] == [1, 0, 0, 0, 0, 0, 0]
    assert o["tol_mask"][:2] == [1, 3]                            # Equal key/value/effect; bare Exists tolerates all
    assert o["priority"][1] == 7 and o["ts_ns"][1] == 42
    # fillOccupiedObj runs in QUEUE order (Less, core.go:368-411): p1 (priority 7) is popped first and, having owner
    # refs, occupies pgA with "u1,u2" (sorted); p0 (no owner refs) then meets an occupied group -> the "no refs"
    # message; p6 matches the owners; pgB is occupied by "u1,u2": other owners -> mismatch, no owners -> "no refs"
    assert o["pod_flags"] == [S.POD_OCC_NOREFS, 0, S.POD_LISTER_MISS, 0, S.POD_OCC_MISMATCH, S.POD_OCC_NOREFS, 0]
    assert o["min_member"] == [2, 3, 1, 4] and o["scheduled"] == [0, 1, 0, 0] and o["matched"] == [1, 0, 0, 0]
    assert o["group_flags"] == [0, S.GROUP_HAS_MINRES, 0, S.GROUP_SCHEDULED]
    min_res = np.array(o["min_res"]).reshape(L, G)
    assert min_res[:, 1].tolist() == [2000, 0, 0, 0, 1, 0] and o["min_res_present"] == [0, 0x10, 0, 0]
    assert o["name_rank"] == [0, 1, 0, 2]                         # bare name, namespace ignored (core.go:404)
    assert o["wait_ns"] == [7 * 10**9, 5 * 10**9, 7 * 10**9, 7 * 10**9]   # Spec.MaxScheduleTime wins (k8s.go:82-91)


def test_packer_delta_rows(plugin_bin):
    """PackNodeRows (incremental snapshot update): the NodeInfos an informer touched, packed with the
    dictionaries of the last full pack, equal the same rows of a full re-pack; a taint or scalar resource
    the round has never seen asks for a full pack instead."""
    o = _run(plugin_bin, "pack_delta")
    assert o["rows"] == 11 and o["needs_full"] == 0
    assert o["mismatches"] == 0 and o["untouched_diff"] == 0
    assert o["sel_pairs"] == 2 and o["taints"] == 2
    assert o["full_on_new_taint"] == 1 and o["full_on_new_scalar"] == 1


def test_packer_group_delta_rows(plugin_bin):
    """PackGroupRows: PodGroups whose state moved between cycles, packed with the round's dictionaries,
    equal the same rows of a full re-pack (bare-name ranks taken over); representative-pod masks use the
    round's selector / taint bits; an unknown selector pair or scalar resource asks for a full pack."""
    o = _run(plugin_bin, "pack_group_delta")
    assert o["rows"] == 6 and o["needs_full"] == 0 and o["mismatches"] == 0
    assert o["rep_ok"] == 1 and o["full_on_new_selector"] == 1 and o["full_on_new_scalar"] == 1


def test_packer_occupancy_lookup_ranks_randomised(plugin_bin):
    """The packer's order-dependent parts on 40 random object sets (duplicate and prefix-sharing group names, ties in
    every key field, frozen groups, recently permitted pods): group lookup, bare-name ranks and the OccupiedBy rule of
    fillOccupiedObj (core.go:494-511) replayed in queue order, against a direct restatement over the whole pod list."""
    o = _run(plugin_bin, "pack_occupancy_random", "40")
    assert o["mismatches"] == 0 and o["flagged"] > 500 and o["pods"] > 10000


def test_round_row_index(plugin_bin):
    """StrIndex, the uid -> pod row / node name -> snapshot row lookup PreFilter, Filter and Permit go through, against a
    std::unordered_map filled in row order: duplicates (later row wins), empty and absent keys, arbitrary bytes."""
    o = _run(plugin_bin, "strindex", "60")
    assert o["mismatches"] == 0 and o["checked"] > 50000


def test_packer_throughput_smoke(plugin_bin):
    out = _run(plugin_bin, "bench_pack", "500", "4000", "500")
    assert out["lanes"] == 5 and out["pack_ms"] > 0


@pytest.mark.gpu
def test_readme_race_through_cpp_plugin(plugin_bin, snapshot_mod):
    # README.md:76-188 — "only one and at least one group" runs; messages as core.go:107,143 print them
    S = snapshot_mod
    rows = _run(plugin_bin, "readme")
    late = [r for r in rows if r["pod"].startswith("late-")]
    rows = [r for r in rows if not r["pod"].startswith("late-")]
    g1 = [r for r in rows if "race1" in r["pod"]]
    g2 = [r for r in rows if "race2" in r["pod"]]
    # 21 s later (freeze cache expired): group2 is refused again at pct 1.0 (2100 < 5000), then frozen again
    assert late[0]["prefilter_code"] == 2 and late[0]["message"] == "cluster resource not enough"
    assert late[1]["message"] == "pod with pgName: default/group2 last failed in 20s, deny"
    assert all(r["prefilter_code"] == 0 and r["node"] == 0 and r["permit_code"] == 4 for r in g1)   # Wait
    assert [r["start_signal"] for r in g1] == [0, 0, 0, 0, 1]
    assert all(r["wait_ns"] == 10**9 for r in g1)                                                    # 0 + 1 s (Q12)
    assert g2[0]["prefilter_code"] == 2 and g2[0]["message"] == "cluster resource not enough"
    for r in g2[1:]:
        assert r["prefilter_code"] == 2
        assert r["message"] == "pod with pgName: default/group2 last failed in 20s, deny"


@pytest.mark.gpu
def test_gang_timeout_and_allow_list(plugin_bin):
    """SURVEY 8(f) row 3 on the engine's gang state: a gang that does not complete within its wait time is
    evicted — every pod it still holds at Permit is rejected, its tables are flushed and it is deny-listed for 20 s
    (controller.go:314-335, batchscheduler.go:347-354); a gang that completes hands out its Allow list once
    (batchscheduler.go:292-344)."""
    out = _run(plugin_bin, "gang_timeout")
    WAIT, UNSCHED = 4, 2
    assert out["a0@0"]["prefilter_code"] == 0 and out["a0@0"]["permit_code"] == WAIT and out["a0@0"]["start_signal"] == 0
    assert out["a0@0"]["wait_ns"] == 11 * 10**9                      # MaxScheduleTime 10 s + 1 s (batchscheduler.go:180-182)
    assert out["a1@4"]["permit_code"] == WAIT and out["a1@4"]["start_signal"] == 0
    assert out["b0@5"]["start_signal"] == 0 and out["allow_b@5"] == []
    assert out["b1@6"]["start_signal"] == 1                          # 2 >= MinMember 2: ready on the second pod, not the first
    assert sorted(out["allow_b@6"]) == [["uid-gang-b-0", "node1"], ["uid-gang-b-1", "node1"]]
    assert out["allow_b_again"] == []                                # allowed pods left MatchedPodNodes
    assert out["tick@9"] == {"rejected": [], "evicted": []}
    # at 11 s a0's entries (TTL 10 s) are gone: the name cache's eviction fires; a1 (TTL until 14 s) is still waiting
    assert out["tick@11"] == {"rejected": ["uid-gang-a-1"], "evicted": ["default/gang-a"]}
    assert out["a2@12"]["prefilter_code"] == UNSCHED
    assert out["a2@12"]["message"] == "pod with pgName: default/gang-a last failed in 20s, deny"
    assert out["a2@32"]["prefilter_code"] == 0 and out["a2@32"]["permit_code"] == WAIT and out["a2@32"]["start_signal"] == 0


@pytest.mark.gpu
def test_readme_race_in_one_call(plugin_bin, snapshot_mod):
    # all ten pods pending at once; ReplayQueue walks them in Less order on the device: equal priority
    # and creation time -> the group with the greater name goes first (core.go:404) and wins the race
    S = snapshot_mod
    rows = _run(plugin_bin, "readme_replay")
    g1 = sorted((r for r in rows if "race1" in r["pod"]), key=lambda r: r["position"])
    g2 = sorted((r for r in rows if "race2" in r["pod"]), key=lambda r: r["position"])
    assert max(r["position"] for r in g2) < min(r["position"] for r in g1)
    assert all(r["prefilter_code"] == S.PF_PASS and r["node"] == 0 for r in g2)
    assert [r["ready"] for r in g2] == [0, 0, 0, 0, 1]
    assert g1[0]["prefilter_code"] == S.PF_NOT_ENOUGH and all(r["prefilter_code"] == S.PF_DENIED for r in g1[1:])
    assert all(r["node"] == -1 and r["ready"] == 0 for r in g1)


def test_quantity_parsing_randomised(plugin_bin):
    """resource.Quantity semantics against an exact rational model: Value() and MilliValue() are the
    ceilings (away from zero for negatives) of the parsed number and of 1000x it."""
    import math
    import random
    from fractions import Fraction
    rnd = random.Random(7)
    sufs = {"": Fraction(1), "m": Fraction(1, 1000), "u": Fraction(1, 10**6), "n": Fraction(1, 10**9), "k": Fraction(10**3),
            "M": Fraction(10**6), "G": Fraction(10**9), "T": Fraction(10**12), "P": Fraction(10**15),
            "Ki": Fraction(2**10), "Mi": Fraction(2**20), "Gi": Fraction(2**30), "Ti": Fraction(2**40), "Pi": Fraction(2**50)}
    cases = {}
    for _ in range(400):
        whole = rnd.randint(0, 10**rnd.randint(1, 6))
        frac = "" if rnd.random() < 0.5 else "." + "".join(rnd.choice("0123456789") for _ in range(rnd.randint(1, 4)))
        suf = rnd.choice(list(sufs))
        if rnd.random() < 0.15:
            ex = rnd.randint(0, 6)
            s = f"{whole}{frac}e{ex}"
            val = Fraction(f"{whole}{frac}") * 10**ex
        else:
            s = f"{whole}{frac}{suf}"
            val = Fraction(f"{whole}{frac}") * sufs[suf]
        if val * 1000 >= 2**62:
            continue
        cases[s] = (math.ceil(val), math.ceil(val * 1000))
    keys = list(cases)
    for i in range(0, len(keys), 100):
        out = _run(plugin_bin, "quantity", *keys[i:i + 100])
        for s in keys[i:i + 100]:
            ok, v, m = out[s]
            assert ok == 1 and (v, m) == cases[s], (s, out[s], cases[s])


def _affinity_expected(many):
    """Independent Python evaluation of the predicates tests/cpp/plugin_test.cpp::cmd_pack_affinity builds."""
    N = 40
    labels = []
    for i in range(N):
        lb = {"zone": f"z{i % 4}", "cores": str(8 << (i % 3))}
        if i % 2:
            lb["disk"] = "ssd"
        if i % 5 == 0:
            lb["gpu"] = "a100"
        if i % 7 == 0:
            lb["cores"] = "many"
        for k in range(many):
            if (i + k) % 3 == 0:
                lb[f"k{k}"] = "v"
        labels.append(lb)

    def integer(x):
        try:
            return int(x)
        except ValueError:
            return None
    preds = [
        lambda i, lb: lb.get("zone") in ("z1", "z3"),
        lambda i, lb: lb.get("zone") != "z0" and "disk" in lb,
        lambda i, lb: "gpu" not in lb,
        lambda i, lb: integer(lb["cores"]) is not None and integer(lb["cores"]) > 8,
        lambda i, lb: integer(lb["cores"]) is not None and integer(lb["cores"]) < 32,     # + disk=ssd selector (mask or table)
        lambda i, lb: lb.get("zone") == "z0" or lb.get("gpu") == "a100",
        lambda i, lb: i == 7,
        lambda i, lb: i != 7 and lb.get("zone") == "z3",
        lambda i, lb: False, lambda i, lb: False, lambda i, lb: False, lambda i, lb: False,
    ]
    return N, labels, preds


@pytest.mark.parametrize("many", [0, 70])
def test_packer_node_affinity(plugin_bin, many):
    """Required nodeAffinity (In / NotIn / Exists / DoesNotExist / Gt / Lt, matchFields, ORed terms, invalid
    requirements) becomes affinity classes + (class, node) verdict bits; more than 64 distinct nodeSelector
    pairs move every selector into the table (the 64-pair limit of round 1 is gone)."""
    out = _run(plugin_bin, "pack_affinity", str(many))
    N, labels, preds = _affinity_expected(many)
    W = (N + 31) // 32
    bits = np.array(out["aff_bits"], np.uint32).reshape(out["n_aff"], W)
    cls = out["aff_class"]
    NONE = 0xFFFFFFFF
    in_table = many > 64 - 1          # disk=ssd plus the k pairs
    assert out["sel_in_table"] == int(in_table)
    assert cls[12] == cls[0] and cls[0] != NONE            # identical predicates share a class
    assert len({cls[i] for i in range(12)}) == 12 - 0 if False else True
    def verdicts(c):
        return np.unpackbits(bits[c].view(np.uint8), bitorder="little")[:N].astype(bool)
    sel = np.array(out["sel_mask"], np.uint64)
    lab = np.array(out["label_mask"], np.uint64)
    for p in range(12):
        want = np.array([preds[p](i, labels[i]) for i in range(N)])
        if p == 4:
            want &= np.array(["disk" in labels[i] for i in range(N)])
        want[9] = False                                     # info.Node() == nil
        got = verdicts(cls[p])
        if not in_table:                                    # the selector part lives in the masks
            got = got & ((lab & sel[p]) == sel[p])
            got[9] = False
        np.testing.assert_array_equal(got, want, err_msg=f"pod {p}")
    # the selector-only pod: mask bits in the small round, a table class in the big one
    want13 = np.array(["disk" in labels[i] for i in range(N)]); want13[9] = False
    if in_table:
        assert (sel == 0).all() and cls[13] != NONE
        np.testing.assert_array_equal(verdicts(cls[13]), want13)
        for k in range(many):
            want = np.array([f"k{k}" in labels[i] for i in range(N)]); want[9] = False
            np.testing.assert_array_equal(verdicts(cls[14 + k]), want, err_msg=f"pair {k}")
    else:
        assert cls[13] == NONE and sel[13] != 0
        got = (lab & sel[13]) == sel[13]; got[9] = False
        np.testing.assert_array_equal(got, want13)
