"""CPU: BatchSchedulingPlugin::PackPreferences (tests/cpp/plugin_node_priority_test.cpp) against an independent
evaluation of the same objects written here from kube-scheduler v1.17's taint_toleration.go, node_affinity.go,
ToleratesTaint and NodeSelectorRequirementsAsSelector [upstream, from memory]: the PreferNoSchedule dictionary, each
pod's tolerated bits (only tolerations with an empty or PreferNoSchedule effect), the class of each pod (deduplicated,
PREF_NONE without a term of non-zero weight) and the class x node weights (every operator, empty expressions and
match_fields matching nothing, weight 0 skipped, an invalid requirement counting 0), and the 64-taint limit."""
import json
import subprocess

import pytest

import native

PREF_NONE = 0xFFFFFFFF


@pytest.fixture(scope="module")
def packed():
    return json.loads(subprocess.check_output([native.cpp_program("plugin_node_priority_test")], text=True))


def tolerates(tol, taint):
    key, op, value, effect = tol
    if effect and effect != taint[2]:
        return False
    if key and key != taint[0]:
        return False
    if op in ("", "Equal"):
        return value == taint[1]
    return op == "Exists"


def requirement(r, labels):
    """(valid, matches) of one label requirement."""
    key, op, values = r
    has = key in labels
    if op in ("In", "NotIn"):
        if not values:
            return False, False
        return True, (has and labels[key] in values) if op == "In" else (not has or labels[key] not in values)
    if op in ("Exists", "DoesNotExist"):
        if values:
            return False, False
        return True, has if op == "Exists" else not has
    if op in ("Gt", "Lt"):
        try:
            bound = int(values[0]) if len(values) == 1 else None
        except ValueError:
            bound = None
        if bound is None:
            return False, False
        try:
            v = int(labels[key]) if has else None
        except ValueError:
            v = None
        return True, v is not None and (v > bound if op == "Gt" else v < bound)
    return False, False


def term_matches(exprs, labels):
    if not exprs:
        return False   # labels.Nothing()
    for r in exprs:
        valid, ok = requirement(r, labels)
        if not valid or not ok:
            return False
    return True


def test_dictionary_and_node_bits(packed):
    want = []
    for nd in packed["nodes"]:
        for k, v, e in nd["taints"]:
            if e == "PreferNoSchedule" and [k, v] not in want:
                want.append([k, v])
    assert packed["dict"] == want
    for i, nd in enumerate(packed["nodes"]):
        bits = sum(1 << want.index([k, v]) for k, v, e in nd["taints"] if e == "PreferNoSchedule")
        assert packed["prefer_taints"][i] == bits, i


def test_tolerated_bits(packed):
    d = packed["dict"]
    for p, pod in enumerate(packed["pods"]):
        tols = [t for t in pod["tolerations"] if t[3] in ("", "PreferNoSchedule")]
        bits = sum(1 << b for b, (k, v) in enumerate(d) if any(tolerates(t, (k, v, "PreferNoSchedule")) for t in tols))
        assert packed["prefer_tol"][p] == bits, p
    # spot checks of the branches: NoSchedule-only toleration does not count; Exists with an empty key takes every
    # bit; an empty operator means Equal
    assert packed["prefer_tol"][1] == 1 << d.index(["k1", "v1"])
    assert packed["prefer_tol"][2] == (1 << len(d)) - 1 and packed["prefer_tol"][8] == (1 << len(d)) - 1
    assert packed["prefer_tol"][3] == sum(1 << d.index(x) for x in (["k1", "v1"], ["k1", "v2"], ["k4", "z"]))
    assert packed["prefer_tol"][0] == 0


def test_classes_and_weights(packed):
    sigs, want_class = [], []
    for pod in packed["pods"]:
        terms = [(w, json.dumps(e)) for w, e, _ in pod["preferred"] if w != 0]
        if not terms:
            want_class.append(PREF_NONE)
            continue
        if terms not in sigs:
            sigs.append(terms)
        want_class.append(sigs.index(terms))
    assert packed["pref_class"] == want_class
    assert want_class[4] == want_class[5] != PREF_NONE      # the same terms share a class
    assert want_class[7] == PREF_NONE and want_class[0] == PREF_NONE
    assert len(packed["pref_weights"]) == len(sigs) == 3
    for c in range(len(sigs)):
        pod = packed["pods"][want_class.index(c)]
        for i, nd in enumerate(packed["nodes"]):
            w = sum(t[0] for t in pod["preferred"] if t[0] != 0 and term_matches(t[1], nd["labels"]))
            assert packed["pref_weights"][c][i] == w, (c, i)
    # the mixed class by hand: zone In a (10), gen Gt 6 (5), rack NotIn 1 + gen DoesNotExist (2); the match_fields
    # term, the invalid zone In () and the weight-0 term count nothing
    assert packed["pref_weights"][want_class[4]] == [10, 5, 12, 0, 2, 15]
    # gen Lt 7 (4) fails on "abc" (not an integer) and on 10; zone Exists (9)
    assert packed["pref_weights"][want_class[6]] == [13, 9, 9, 9, 0, 9]
    # rack Gt "x" is invalid: the term counts 0, the other still counts
    assert packed["pref_weights"][want_class[8]] == [10, 0, 10, 0, 0, 10]


def test_taint_limit(packed):
    assert packed["packs_64"] == 64
    assert packed["packs_65"] == -1
