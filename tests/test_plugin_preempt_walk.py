"""PreemptQueue through the C++ plugin (tests/cpp/plugin_preempt_walk_test.cpp) on the GPU: the two-node scenario of
tests/preempt_walk_cases.py ("gang_rolls_back") in a round, with the group's pods around an online pod in the queue."""
import json
import subprocess

import pytest

import native

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def out():
    return json.loads(subprocess.check_output([native.cpp_program("plugin_preempt_walk_test"), "walk"], text=True))


def test_queue_covers_preempt_all(out):
    assert out["bound"] == 4
    assert out["all"]["ok"] and out["queue"]["ok"]
    assert sorted(e[0] for e in out["queue"]["entries"]) == sorted(e[0] for e in out["all"]["entries"]) == \
        ["uid-g1", "uid-g2", "uid-g3", "uid-q"]
    victims = [v for e in out["queue"]["entries"] for v in e[2]]
    assert len(victims) == len(set(victims)) > 0
    first = out["queue"]["entries"][0]
    assert out["first"] == first[1:]   # the walk's first step is bs_preempt's answer
    # PreemptAll answers each pod alone: every one gets node-0 and its two victims (node-1's first victim d has the
    # higher priority)
    for uid, node, vs in out["all"]["entries"]:
        assert [node, vs] == ["node-0", ["uid-a", "uid-b"]], uid


@pytest.mark.parametrize("key", ["queue", "gang"])
def test_queue_equals_the_direct_walk(out, key):
    """PreemptQueue equals bs_preempt_walk called on the same rows in the same order."""
    assert out[key + "_direct"]["rc"] == 0
    assert out[key]["entries"] == out[key + "_direct"]["entries"]


def test_queue_without_gang_units(out):
    """In queue order, the first preemptor takes node-0 and the second node-1; the other two find no node."""
    got = [e[1:] for e in out["queue"]["entries"]]
    assert got == [["node-0", ["uid-a", "uid-b"]], ["node-1", ["uid-d", "uid-c"]], ["", []], ["", []]]


def test_gang_units(out):
    g = out["gang"]
    assert g["ok"]
    uids = [e[0] for e in g["entries"]]
    k = uids.index("uid-g1")
    assert uids[k:k + 3] == ["uid-g1", "uid-g2", "uid-g3"]   # the group is walked as one unit
    got = {e[0]: e[1:] for e in g["entries"]}
    assert got["uid-q"] == ["node-0", ["uid-a", "uid-b"]]
    for m in ("uid-g1", "uid-g2", "uid-g3"):
        assert got[m] == ["", []]   # the third member finds no node: the unit rolls back


def test_mixed_priority_group(out):
    assert not out["mixed_gang"]["ok"] and "ns/g" in out["mixed_gang"]["message"]
    assert out["mixed_queue"]["ok"]
