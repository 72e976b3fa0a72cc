"""The snapshot packer's row encoding (batch-scheduler_b200/csrc/plugin.cpp) on CPU: the full pack and the incremental
row re-packs (PackNodeRows / PackGroupRows) must give every object the same row."""
import json
import subprocess

import native


def test_packer_row_reencode_randomised():
    """Every node and group row of a full pack of 40 random object sets, re-encoded by PackNodeRows / PackGroupRows
    under that pack's dictionaries, equals the full pack's row in every column (affinity verdicts, representative-pod
    masks and classes, ranks and wait times included). A NoSchedule / NoExecute taint, a scalar resource, a selector
    pair or an affinity predicate the round does not hold asks for a full pack; a PreferNoSchedule taint or a resource
    name Resource.Add ignores does not."""
    o = json.loads(subprocess.check_output([native.cpp_program("pack_rows_test"), "pack_rows_random", "40"], text=True))
    assert o["mismatches"] == 0 and o["needs_full"] == 0
    assert o["node_rows"] > 10000 and o["group_rows"] > 2000
    assert o["triggers"] == 40 * 10 and o["fired"] == o["triggers"] and o["false_full"] == 0
    cover = o["cover"]
    for k in ("nil", "no_node", "taints_err", "unschedulable", "NoSchedule", "NoExecute", "PreferNoSchedule",
              "lanes_ge_6", "ignored_name", "min_res", "no_min_res", "rep_sel", "rep_tol", "rep_aff", "aff_classes",
              "sel_in_masks", "sel_in_table"):
        assert cover.get(k, 0) > 0, k
