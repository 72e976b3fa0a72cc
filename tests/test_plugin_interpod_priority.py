"""CPU: BatchSchedulingPlugin::PackInterPodAffinity (tests/cpp/plugin_interpod_priority_test.cpp) against the packing
rules restated over the same objects in tests/pyref_interpod_priority.py (pack): the topology keys and each key's
values in order of first appearance, the term dictionary (resolved namespaces, converted selector and key; a nil
selector kept apart from an empty one; empty keys left out), the bound pods and their classes, each pending pod's
class, at hard weights 0, 1 and 100; the invalid-selector rule (a pending pod's own invalid term takes its class away,
a bound pod's takes every pending pod's); the 64-key limit; and the range of SetHardPodAffinityWeight."""
import json
import subprocess

import pytest

import native
import pyref_interpod_priority as pyi


@pytest.fixture(scope="module")
def out():
    return json.loads(subprocess.check_output([native.cpp_program("plugin_interpod_priority_test")], text=True))


def _term(t):
    sel = None
    if t["selector"] is not None:
        sel = pyi.Selector(dict(t["selector"]["match_labels"]),
                           [(k, op, list(v)) for k, op, v in t["selector"]["match_expressions"]])
    return pyi.Term(sel, tuple(t["namespaces"]), t["key"])


def _pod(o, node=None):
    return pyi.PodObj(o["ns"], dict(o["labels"]), [_term(t) for t in o["required"]],
                      [(w, _term(t)) for w, t in o["preferred"]], [(w, _term(t)) for w, t in o["anti"]],
                      o["terminating"], node)


def _objects(sc):
    labels = [n["labels"] for n in sc["nodes"]]
    bound = [_pod(b, i) for i, n in enumerate(sc["nodes"]) for b in n["pods"]]
    return [_pod(p) for p in sc["pods"]], bound, labels


@pytest.mark.parametrize("scenario", range(3))
@pytest.mark.parametrize("hard", [0, 1, 100])
def test_packing_matches_the_rules(out, scenario, hard):
    sc = out["scenarios"][scenario]
    pending, bound, labels = _objects(sc)
    want = pyi.pack(pending, bound, labels, hard)
    got = sc["packed"][str(hard)]
    nv, topo, term_key, bound_node, bound_class, bcl = want["node"]
    pod_class, pcl = want["pods"]
    assert got["keys"] == want["keys"]
    assert got["values"] == want["values"]
    assert got["n_values"] == nv
    assert got["topo"] == [v for row in topo for v in row]
    assert got["term_key"] == term_key
    assert got["bound_node"] == bound_node
    assert got["bound_class"] == bound_class
    assert got["bound_classes"] == [list(x) for x in bcl]
    assert got["pod_class"] == pod_class
    assert got["pod_classes"] == [list(x) for x in pcl]


def test_scenarios_cover_the_rules(out):
    """The objects reach what the rules distinguish: classes on both sides, both signs, every kind of term, and the
    invalid-selector rule in both directions."""
    scs = out["scenarios"]
    p0 = scs[0]["packed"]["1"]
    assert any(c != pyi.IPA_NONE for c in p0["pod_class"]) and any(c != pyi.IPA_NONE for c in p0["bound_class"])
    own = p0["bound_classes"][2] + p0["pod_classes"][2]
    assert min(own) < 0 < max(own) and 1 in p0["pod_classes"][3] and 1 in p0["bound_classes"][3]
    pods = [p for sc in scs for n in sc["nodes"] for p in n["pods"]] + [p for sc in scs for p in sc["pods"]]
    terms = [t for p in pods for t in p["required"]] + [t for p in pods for _, t in p["preferred"] + p["anti"]]
    assert any(t["selector"] is None for t in terms) and any(t["key"] == "" for t in terms)
    assert any(t["namespaces"] for t in terms) and any(not t["namespaces"] for t in terms)
    assert any(t["selector"] == {"match_labels": {}, "match_expressions": []} for t in terms)
    # scenario 1: pending pod 4's own invalid term; scenario 2: a bound pod's too
    assert scs[1]["packed"]["1"]["pod_class"][4] == pyi.IPA_NONE
    assert any(c != pyi.IPA_NONE for c in scs[1]["packed"]["1"]["pod_class"])
    assert set(scs[2]["packed"]["1"]["pod_class"]) == {pyi.IPA_NONE}
    # the hard weight reaches the bound classes' own weights
    assert scs[0]["packed"]["0"]["bound_classes"] != scs[0]["packed"]["100"]["bound_classes"]


def test_limits(out):
    assert out["packs_64"] == 64 and out["packs_65"] == -1
    assert out["hard_weight_ok"] == [False, True, True, False]
