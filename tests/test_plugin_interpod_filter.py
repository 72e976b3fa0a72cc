"""BatchSchedulingPlugin and the MatchInterPodAffinity filter (tests/cpp/plugin_interpod_filter_test.cpp).

CPU: PackInterPodFilter's columns, evaluated by tests/interpod_filter_ref.c, give on every node the verdict that
tests/pyref_interpod_filter.py computes independently from the same objects with upstream's topology-pair maps; the
scenarios reach every role, both self_match values, the first-pod exception, nil / empty / invalid selectors, an empty
key and a NodeInfo without a Node.  GPU: a plugin round with SetInterPodAffinityFilter(true) gives each pod's
InterPodReasonCounts and FitError text as restated from those verdicts, and ReplayQueue, Preempt, PreemptAll and
PreemptQueue refuse to run until the filter is off."""
import json
import subprocess
from importlib import import_module

import numpy as np
import pytest

import interpod_filter_ref as fr
import native
import pyref_interpod_filter as py

_CODE = {None: fr.PASS, "E": fr.FAIL_E, "A": fr.FAIL_A, "N": fr.FAIL_N}


def _run(*args):
    return json.loads(subprocess.check_output([native.cpp_program("plugin_interpod_filter_test"), *args], text=True))


@pytest.fixture(scope="module")
def out():
    return _run()


def _term(t):
    sel = t["selector"]
    return py.Term(py.INVALID if sel == "invalid" else sel, t["key"], list(t["namespaces"]))


def _pod(o, node=None):
    return py.Pod(o["name"], o["ns"], dict(o["labels"]), node, [_term(t) for t in o["affinity"]],
                  [_term(t) for t in o["anti"]], o["terminating"])


def _objects(sc):
    nodes = {n["name"]: (dict(n["labels"]) if n["has_node"] else {}) for n in sc["nodes"]}
    # pods of a NodeInfo without a Node contribute nothing: they are left out, as upstream's guard leaves them
    existing = [_pod(b, n["name"]) for n in sc["nodes"] if n["has_node"] for b in n["pods"]]
    return nodes, existing, [_pod(p) for p in sc["pods"]]


def _columns(sc):
    k = sc["packed"]
    node = (k["n_values"], np.array(k["topo"], np.uint32), k["term_key"], k["bound_node"], k["bound_class"],
            tuple(k["bound_classes"]))
    return node, (k["pod_class"], tuple(k["pod_classes"]))


def _want(sc):
    nodes, existing, pending = _objects(sc)
    return np.array([[_CODE[py.verdict(p, n, nodes, existing)] for n in nodes] for p in pending], np.uint8)


@pytest.mark.parametrize("scenario", range(3))
def test_packing_gives_the_verdicts_of_the_objects(out, scenario):
    sc = out["scenarios"][scenario]
    got = fr.verdicts(_columns(sc), len(sc["nodes"]))
    np.testing.assert_array_equal(got, _want(sc))


def test_scenarios_cover_the_rules(out):
    scs = out["scenarios"]
    roles = {r for sc in scs for r in sc["packed"]["pod_classes"][2]}
    assert roles == {py.AFFINITY, py.ANTI, py.EXISTING}
    assert {s for sc in scs for s in sc["packed"]["pod_classes"][3]} == {0, 1}
    v = np.concatenate([_want(sc).ravel() for sc in scs])
    assert set(np.unique(v).tolist()) == {fr.PASS, fr.FAIL_E, fr.FAIL_A, fr.FAIL_N}
    terms = [t for sc in scs for p in sc["pods"] + [b for n in sc["nodes"] for b in n["pods"]]
             for t in p["affinity"] + p["anti"]]
    sels = [t["selector"] for t in terms]
    assert None in sels and {} in sels and "invalid" in sels and any(t["key"] == "" for t in terms)
    assert any(t["namespaces"] for t in terms) and any(not n["has_node"] and n["pods"] for sc in scs for n in sc["nodes"])
    # the first-pod exception: a pod whose affinity pair map is empty still passes a node
    assert any(p.affinity and not py.getTPMapMatchingIncomingAffinityAntiAffinity(p, existing, nodes)[0] and
               py.verdict(p, n, nodes, existing) is None
               for nodes, existing, pending in map(_objects, scs) for p in pending for n in nodes)


@pytest.mark.gpu
def test_plugin_round(pkg):
    o = _run("gpu")
    sc = o["scenarios"][0]
    v = _want(sc)
    has_node = np.array([n["has_node"] for n in sc["nodes"]])
    eng = import_module("batch-scheduler_b200.engine")
    for k, r in enumerate(sc["round"]):
        # every node with a Node fits every pod but for the filter: the lane rows count only the Node-less one
        assert r["reasons"][:4] == [0, int((~has_node).sum()), 0, 0] and not any(r["reasons"][4:])
        comp = fr.companion_rows(v[k:k + 1], has_node[None, :])[0]
        assert r["interpod"] == comp.tolist()
        fits = int(((v[k] == fr.PASS) & has_node).sum())
        want = eng.format_fit_error(r["reasons"], sc["lanes"], len(sc["nodes"]), interpod=comp) if fits == 0 else ""
        assert r["fit_error"] == want
    assert any(r["fit_error"] for r in sc["round"]) and any(not r["fit_error"] for r in sc["round"])
    assert sc["refused"] == [True, True, True, True]
    assert sc["replay_after_off"] and sc["interpod_after_off"] == []
