"""PodDisruptionBudgets in preemption through the C++ plugin (tests/cpp/plugin_preempt_pdb_test.cpp): PackBoundPods'
classification on the CPU, and on the GPU the hand-built cases 1-4 of tests/pdb_cases.py through Preempt, PreemptAll
and a direct bs_preempt call, and when SetPodDisruptionBudgets takes effect."""
import json
import subprocess

import pytest

import native

VIOLATING, LOCKED = 0x02, 0x01


@pytest.fixture(scope="module")
def binary():
    return native.cpp_program("plugin_preempt_pdb_test")


def _run(binary, mode):
    return json.loads(subprocess.check_output([binary, mode], text=True))


def test_pack_classification(binary):
    o = _run(binary, "pack")
    assert o["ok"]
    assert o["with"] == {
        "plain": 0,           # no budget selects it
        "other-ns": 0,        # the budget selecting it is in another namespace
        "no-labels": 0,       # a pod without labels matches no budget ...
        "labelled": VIOLATING,   # ... while the same budget matches a labelled pod of its namespace
        "nil-sel": 0,         # a nil selector matches nothing
        "bad-sel": 0,         # selectors that fail LabelSelectorAsSelector are skipped
        "allow-1": 0,         # the budget still allows a disruption
        "allow-0": VIOLATING,
        "allow-neg": VIOLATING,
        "two": VIOLATING,     # two budgets match, one of them allows nothing
        "locked": VIOLATING | LOCKED,
    }   # the empty selector of namespace "ns" would mark every pod there if it matched
    assert o["without"] == {k: (LOCKED if k == "locked" else 0) for k in o["with"]}


WANT = {   # tests/pdb_cases.py cases 1-4, as the plugin names the nodes and pods
    "1": ["node-0", ["uid-b"]],
    "2": ["node-1", ["uid-w"]],
    "3": ["node-0", ["uid-v", "uid-w"]],
    "4": ["node-1", ["uid-v1", "uid-w1"]],
}


@pytest.mark.gpu
def test_cases_through_the_plugin(binary):
    o = _run(binary, "cases")
    assert set(o) == set(WANT)
    for c, want in WANT.items():
        assert o[c]["preempt"] == want, c
        assert o[c]["all"] == want, c
        assert o[c]["direct"] == want, c


@pytest.mark.gpu
def test_set_budgets_takes_effect_when_the_table_is_packed(binary):
    o = _run(binary, "setter")
    plain, budgeted = ["node-0", ["uid-v"]], ["node-1", ["uid-w"]]
    assert o["none"] == plain
    assert o["set"] == plain               # the uploaded table is unchanged until it is packed again
    assert o["update_nodes"] == budgeted   # UpdateNodes packs it again
    assert o["cleared_begin_round"] == plain
    assert o["set_begin_round"] == budgeted
