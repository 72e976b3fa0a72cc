"""BatchSchedulingPlugin and the PodFitsHostPorts filter (tests/cpp/plugin_host_ports_test.cpp).

CPU: PackHostPorts' columns equal tests/pyref_host_ports.py's independent pack of the same objects (the dictionary's
order and pruning included), tests/host_ports_ref.c over them gives the verdicts the object restatement gives, and 65
distinct wanted entries are refused while 64 pack.  GPU: a plugin round with SetHostPortFilter(true) gives each pod's
HostPortReasonCounts and FitError text as restated from those verdicts; the switch repacks on UpdateNodes and
UpdateRound; ReplayQueue runs under the filter and never places a pod on a port it conflicts with; Preempt,
PreemptAll and PreemptQueue refuse to run."""
import json
import subprocess
from importlib import import_module

import numpy as np
import pytest

import host_ports_ref as hr
import native
import pyref_host_ports as py


def _run(*args):
    return json.loads(subprocess.check_output([native.cpp_program("plugin_host_ports_test"), *args], text=True))


@pytest.fixture(scope="module")
def out():
    return _run()


def _ports(lst):
    return [py.Port(hp, ip, proto, cp) for ip, proto, hp, cp in lst]


def _objects(sc):
    nodes = [py.Node(f"node-{i}", _ports(u)) for i, u in enumerate(sc["nodes"])]
    pods = [py.Pod(f"p{k}", _ports(w)) for k, w in enumerate(sc["pods"])]
    return nodes, pods


@pytest.mark.parametrize("scenario", range(3))
def test_packing_matches_the_objects(out, scenario):
    sc = out["scenarios"][scenario]
    nodes, pods = _objects(sc)
    entries, used, want = py.pack(nodes, pods)
    k = sc["packed"]
    assert np.array(k["entries"], np.int64).reshape(-1, 3).tolist() == entries.tolist()
    assert k["used"] == used.tolist() and k["want"] == want.tolist()
    np.testing.assert_array_equal(hr.passes(k["entries"], np.array(k["used"], np.uint64),
                                            np.array(k["want"], np.uint64)), py.verdicts(pods, nodes))


def test_scenarios_cover_the_rules(out):
    allp = [p for sc in out["scenarios"] for grp in (sc["nodes"], sc["pods"]) for lst in grp for p in lst]
    ips = {p[0] for p in allp}
    assert {"", "0.0.0.0", "::"} <= ips and {"", "TCP", "UDP"} <= {p[1] for p in allp}
    assert any(p[2] <= 0 for p in allp)
    v = np.concatenate([py.verdicts(*reversed(_objects(sc))).ravel() for sc in out["scenarios"]])
    assert v.any() and not v.all()


def test_dictionary_limit(out):
    assert out["refuses_65"] and out["packs_64"] and out["entries_64"] == 64


@pytest.mark.gpu
def test_plugin_round(pkg):
    o = _run("gpu")
    sc = o["scenarios"][0]
    nodes, pods = _objects(sc)
    eng = import_module("batch-scheduler_b200.engine")
    N = len(nodes)

    def check(rounds, nodes):
        v = py.verdicts(pods, nodes)
        for k, r in enumerate(rounds):
            # every node fits every pod but for the ports: the lane rows are all zero
            assert not any(r["reasons"])
            cnt = int((~v[k]).sum())
            assert r["host_ports"] == [cnt]
            want = eng.format_fit_error(r["reasons"], sc["lanes"], N, host_ports=[cnt]) if v[k].sum() == 0 else ""
            assert r["fit_error"] == want
        return v
    v = check(sc["round"], nodes)
    assert (~v).any()
    assert sc["update_nodes_ok"] and sc["update_round_ok"]
    full = [py.Node("node-0", _ports(sc["node0_ports"]))] + nodes[1:]
    v2 = check(sc["after_update_nodes"], full)
    wants = np.array([bool(py.triples(p.ports)) for p in pods])
    assert not v2[wants, 0].any() and (v2 != v).any()
    check(sc["after_update_round"], nodes)
    assert sc["refused"] == [True, True, True]
    # the walk: no pod lands on a node whose live ports conflict with its own
    assert sc["replay_runs"]
    live = [list(py.triples(n.used)) for n in nodes]
    for pos, n in enumerate(sc["replay_nodes"]):
        if n < 0:
            continue
        p = pods[sc["queue"][pos]]
        assert py.verdict(p, py.Node("live", [py.Port(t[2], t[0], t[1]) for t in live[n]]))
        live[n] += py.triples(p.ports)
