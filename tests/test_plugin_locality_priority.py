"""CPU: BatchSchedulingPlugin::PackLocality (tests/cpp/plugin_locality_priority_test.cpp) against an independent
evaluation of the same objects written here from kube-scheduler v1.17's image_locality.go and
node_prefer_avoid_pods.go [upstream, from memory]: the image-name normalization, the dictionary of reported names that
some pod's normalized image matches (sizes from the lowest node index, bit rows), the classes (sorted id lists,
deduplicated, repeats kept, IMAGE_NONE without a dictionary image), the avoid dictionary of RC / RS controllers both
listed on a node and controlling a pod, each node's and pod's bits, and the 64-controller limit."""
import json
import subprocess

import pytest

import native
import pyref_locality_priority as pyl

IMAGE_NONE, AVOID_NONE = 0xFFFFFFFF, 0xFF


@pytest.fixture(scope="module")
def packed():
    return json.loads(subprocess.check_output([native.cpp_program("plugin_locality_priority_test")], text=True))


def test_normalization(packed):
    for name, got in packed["normalized"]:
        assert got == pyl.normalized_image_name(name), name
    assert dict(packed["normalized"])["registry:5000/team/app"] == "registry:5000/team/app:latest"


def _expected(o):
    wanted = {pyl.normalized_image_name(im) for pod in o["pods"] for im in pod["images"]}
    names, size, rows = [], [], []
    N = len(o["nodes"])
    for i, nd in enumerate(o["nodes"]):
        for im_names, sz in nd["images"]:
            for nm in im_names:
                if nm not in wanted:
                    continue
                if nm not in names:
                    names.append(nm)
                    size.append(sz)
                    rows.append(set())
                rows[names.index(nm)].add(i)
    classes, cls = [], []
    for pod in o["pods"]:
        ids = sorted(names.index(pyl.normalized_image_name(im)) for im in pod["images"]
                     if pyl.normalized_image_name(im) in names)
        if not ids:
            cls.append(IMAGE_NONE)
            continue
        if ids not in classes:
            classes.append(ids)
        cls.append(classes.index(ids))
    controlling = {tuple(p["controller"]) for p in o["pods"]
                   if p["controller"][0] in ("ReplicationController", "ReplicaSet")}
    ctrls, mask = [], [0] * N
    for i, nd in enumerate(o["nodes"]):
        for c in map(tuple, nd["avoid"]):
            if c not in controlling:
                continue
            if c not in ctrls:
                ctrls.append(c)
            mask[i] |= 1 << ctrls.index(c)
    bits = [ctrls.index(tuple(p["controller"])) if tuple(p["controller"]) in ctrls else AVOID_NONE for p in o["pods"]]
    return names, size, rows, classes, cls, ctrls, mask, bits


def test_dictionary_and_classes(packed):
    o = packed
    names, size, rows, classes, cls, ctrls, mask, bits = _expected(o)
    N = len(o["nodes"])
    W = (N + 31) // 32
    assert o["names"] == names
    assert o["image_size"] == size
    got_rows = [{n for n in range(N) if (o["image_bits"][i * W + n // 32] >> (n % 32)) & 1} for i in range(len(names))]
    assert got_rows == rows
    got_classes = [o["class_images"][o["class_offset"][c]:o["class_offset"][c + 1]]
                   for c in range(len(o["class_offset"]) - 1)]
    assert got_classes == classes
    assert o["image_class"] == cls
    assert [tuple(c) for c in o["controllers"]] == ctrls
    assert o["avoid_mask"] == mask
    assert o["avoid_bit"] == bits


def test_hand_facts(packed):
    """The facts the scenario was built to show, stated directly."""
    o = packed
    names = o["names"]
    assert names[0] == "nginx:latest" and o["image_size"][0] == 100 << 20     # node 0's size, not node 1's 120 MiB
    assert "registry:5000/team/train" not in names                          # reported untagged: no pod matches it
    assert "unused:1" not in names                                          # no pod asks for it
    assert "cuda:latest" in names                                           # pod 7's "cuda" normalized
    assert o["image_class"][2] == o["image_class"][4] != IMAGE_NONE          # same images, other order
    c1 = o["image_class"][1]
    assert o["class_images"][o["class_offset"][c1]:o["class_offset"][c1 + 1]] == [0, 0]   # a repeated image stays
    assert o["image_class"][5] == o["image_class"][6] == IMAGE_NONE         # busybox unreported, no containers
    ctrls = [tuple(c) for c in o["controllers"]]
    assert ("Deployment", "d-1") not in ctrls and ("ReplicaSet", "rs-9") not in ctrls
    assert o["avoid_bit"][2] == o["avoid_bit"][4] == o["avoid_bit"][6] == o["avoid_bit"][7] == AVOID_NONE
    assert o["avoid_bit"][0] == o["avoid_bit"][5] != AVOID_NONE


def test_controller_limit(packed):
    assert packed["packs_64"] == 64
    assert packed["packs_65"] == -1
