"""Preemption through the C++ plugin (tests/cpp/plugin_preempt_test.cpp): the bound-pod packer on the CPU, and a
scripted gang scenario through BatchSchedulingPlugin on the GPU."""
import json
import subprocess

import pytest

import native

LOCKED_MSG = "pod belongs to Scheduled or Running pod group can not be scheduled"


@pytest.fixture(scope="module")
def binary():
    return native.cpp_program("plugin_preempt_test")


def test_pack_bound_pods(binary):
    o = json.loads(subprocess.check_output([binary, "pack"], text=True))
    assert o["ok"] and o["n"] == 5
    assert o["node"] == [0, 0, 1, 1, 1]
    assert o["req"][0] == [1000, 500, 2000, 2000, 2000]   # Requests (1 cpu), not Limits (4 cpus)
    assert o["req"][3] == [0, 0, 0, 0, 0]                  # lane 3 is not removed
    assert o["req"][4] == [1, 0, 0, 0, 0] and o["req_present"] == [16, 0, 0, 0, 0]
    assert o["gid"] == [-1, 0, 1, 2, -2]                   # no label, Pending, Running, Scheduled, not in the cache
    assert o["flags"] == [0, 0, 1, 1, 0]                   # Running and Scheduled lock their pods
    assert o["priority"] == [3, -4, 0, 0, 0] and o["start"] == [7, 8, 9, 9, 9]
    assert "scalar resource" in o["errors"][0] and "bad quantity" in o["errors"][1]


@pytest.mark.gpu
def test_gang_scenario(binary):
    o = json.loads(subprocess.check_output([binary, "gang"], text=True))
    assert o["bound"] == 5
    pre = o["preempt"]
    # online P1: the Running gang is off limits, the Pending gang's node loses to the online pod's lower priority
    assert pre["uid-p1"] == ["node-2", ["uid-online"]]
    # offline P2: kept off node-2 (a lower-priority online pod) and node-1 (Running gang); evicts one Pending pod
    assert pre["uid-p2"] == ["node-0", ["uid-pend-b"]]
    # online P3, zone=a only: may evict a Pending gang's pod, not a Running gang's
    assert pre["uid-p3"] == ["node-0", ["uid-pend-b"]]
    assert o["remove"] == [
        [0, ""], [2, LOCKED_MSG], [0, ""],
        [2, "offline pods p2 are forbidden to preempt online online"], [0, ""], [2, LOCKED_MSG]]
    assert o["all_ok"]
    got = {uid: [node, victims] for uid, node, victims in o["all"]}
    assert {"uid-p1", "uid-p3"} <= set(got) <= {"uid-p1", "uid-p2", "uid-p3"}
    for uid, v in got.items():
        assert v == pre[uid]
    # the Pending gang starts running: after the delta round its pods are locked too
    assert o["after"]["uid-p3"] == ["", []]
    assert o["after"]["uid-p1"] == ["node-2", ["uid-online"]]
    assert o["unknown"] == "error"
