"""Preempt, PreemptAll and PreemptQueue through the C++ plugin under the PodFitsHostPorts filter
(tests/cpp/plugin_preempt_host_ports_test.cpp) on the GPU, against answers restated from the program's objects.

Two nodes of 4 cpus, both full with 2-cpu online pods.  node-0: a (prio 0, start 50, 0.0.0.0:22), b (prio 0, start
100, no port).  node-1: c (prio 0, start 100, 10.0.0.1:22), d (prio 100, start 0, 0.0.0.0:8080).  Pending, 1 cpu and
priority 10 each, in queue order: p (:22 with an empty ip, so 0.0.0.0), q (0.0.0.0:8080), r (0.0.0.0:22).

Filter off, each pod alone: on node-0 a is reprieved and b goes; on node-1 c goes; the two tie up to the start time of
their victims (100 each), so node-0 wins by index.  In the walk p takes node-0 ([b]); q then fits node-0 beside a
without victims; r must evict a on node-0 (start 50) or c on node-1 (start 100), and the later start wins: node-1.

Filter on, each pod alone: a and c hold ports that conflict with :22, so for p and r they are victims for their port;
node-0 evicts a and keeps b, node-1 evicts c, and node-1 wins on c's later start.  q conflicts with d's 8080, which
priority 100 protects: node-1 drops out and q evicts b on node-0 (a is reprieved: 22 does not conflict with 8080).
In the walk p takes node-1 ([c]) and is nominated there with 0.0.0.0:22; q takes node-0 ([b]); r finds node-1's
nominated :22 in its way and evicts a on node-0."""
import json
import subprocess

import pytest

import native

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def out():
    return json.loads(subprocess.check_output([native.cpp_program("plugin_preempt_host_ports_test"), "run"], text=True))


def _entries(res):
    assert res["ok"], res["message"]
    return {uid: [node, victims] for uid, node, victims in res["entries"]}


def test_bound_masks(out):
    """The dictionary holds the wanted entries first, then the used ones that conflict with them; each bound pod's
    mask has the bit of each entry one of its ports equals."""
    pk = out["packed"]
    assert pk["ok"]
    assert pk["entries"] == [["0.0.0.0", "TCP", 22], ["0.0.0.0", "TCP", 8080], ["10.0.0.1", "TCP", 22]]
    assert pk["used"] == [1, 6]
    assert pk["bound"] == [1, 0, 4, 2]   # a, b, c, d


def test_filter_off(out):
    o = out["off"]
    assert _entries(o["all"]) == {"uid-p": ["node-0", ["uid-b"]], "uid-q": ["node-0", ["uid-b"]],
                                  "uid-r": ["node-0", ["uid-b"]]}
    assert _entries(o["queue"]) == {"uid-p": ["node-0", ["uid-b"]], "uid-q": ["node-0", []],
                                    "uid-r": ["node-1", ["uid-c"]]}
    assert o["preempt_r"]["ok"] and [o["preempt_r"]["node"], o["preempt_r"]["victims"]] == ["node-0", ["uid-b"]]


def test_filter_on_in_preemption(out):
    o = out["on"]
    assert _entries(o["all"]) == {"uid-p": ["node-1", ["uid-c"]], "uid-q": ["node-0", ["uid-b"]],
                                  "uid-r": ["node-1", ["uid-c"]]}
    assert [e[0] for e in o["queue"]["entries"]] == ["uid-p", "uid-q", "uid-r"]
    assert _entries(o["queue"]) == {"uid-p": ["node-1", ["uid-c"]], "uid-q": ["node-0", ["uid-b"]],
                                    "uid-r": ["node-0", ["uid-a"]]}
    assert o["preempt_r"]["ok"] and [o["preempt_r"]["node"], o["preempt_r"]["victims"]] == ["node-1", ["uid-c"]]


def test_option_off_refuses(out):
    o = out["refused"]
    for key in ("all", "queue", "preempt_r"):
        assert not o[key]["ok"] and "PodFitsHostPorts" in o[key]["message"], key
