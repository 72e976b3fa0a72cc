"""CPU: BatchSchedulingPlugin::PackSpread (tests/cpp/plugin_spread_priority_test.cpp) against an independent evaluation
of the same objects written here from kube-scheduler v1.17's selector_spreading.go and the Service,
ReplicationController, ReplicaSet and StatefulSet listers [upstream, from memory]: the zone keys (region and zone,
zone only, region only, none) in order of first appearance and the 64-zone limit; each pod's selectors (a nil Service
selector matches nothing and an empty one everything; an empty RC, RS or StatefulSet selector matches nothing; a
selector that fails to convert is skipped; a pod without labels gets no RC, RS or StatefulSet; other namespaces do not
count), ANDed; the classes; and the counts, which skip terminating pods and other namespaces."""
import json
import subprocess

import pytest

import native

SPREAD_NONE, ZONE_NONE = 0xFFFFFFFF, 0xFF
R, Z = "failure-domain.beta.kubernetes.io/region", "failure-domain.beta.kubernetes.io/zone"


@pytest.fixture(scope="module")
def packed():
    return json.loads(subprocess.check_output([native.cpp_program("plugin_spread_priority_test")], text=True))


def _map_sel(m):
    """labels.SelectorFromSet: a function of the labels."""
    return lambda labels: all(labels.get(k) == v for k, v in m.items())


def _label_sel(ls):
    """metav1.LabelSelectorAsSelector of a non-nil selector, or None when a requirement fails to convert."""
    reqs = []
    for key, op, values in ls["match_expressions"]:
        if op in ("In", "NotIn") and not values:
            return None
        if op in ("Exists", "DoesNotExist") and values:
            return None
        if op not in ("In", "NotIn", "Exists", "DoesNotExist"):
            return None
        reqs.append((key, op, frozenset(values)))
    ml = dict(ls["match_labels"])

    def match(labels):
        if any(labels.get(k) != v for k, v in ml.items()):
            return False
        for key, op, values in reqs:
            has = key in labels
            if op == "In" and not (has and labels[key] in values):
                return False
            if op == "NotIn" and has and labels[key] in values:
                return False
            if op == "Exists" and not has:
                return False
            if op == "DoesNotExist" and has:
                return False
        return True
    return match, (frozenset(ml.items()), frozenset(reqs))


def _selectors(o, pod):
    """getSelectors: [(identity, match)] of the pod."""
    out = []
    labels = pod["labels"]
    for ns, sel in o["services"]:
        if ns == pod["ns"] and sel is not None and _map_sel(sel)(labels):
            out.append((("map", frozenset(sel.items())), _map_sel(sel)))
    if labels:   # the RC / RS / StatefulSet listers return an error for a pod without labels
        for ns, sel in o["controllers"]:
            if ns == pod["ns"] and sel and _map_sel(sel)(labels):
                out.append((("map", frozenset(sel.items())), _map_sel(sel)))
        for ns, ls in o["replica_sets"] + o["stateful_sets"]:
            if ns != pod["ns"] or ls is None or (not ls["match_labels"] and not ls["match_expressions"]):
                continue
            conv = _label_sel(ls)
            if conv is not None and conv[0](labels):
                out.append((("ls", conv[1]), conv[0]))
    return out


def _count(pod, sels, node):
    if not sels:
        return 0
    return sum(1 for b in node["pods"] if b["ns"] == pod["ns"] and not b["terminating"]
               and all(m(b["labels"]) for _, m in sels))


def test_zones(packed):
    o = packed
    keys, zone = [], []
    for nd in o["nodes"]:
        r, z = nd["labels"].get(R, ""), nd["labels"].get(Z, "")
        if not r and not z:
            zone.append(ZONE_NONE)
            continue
        k = r + ":\x00:" + z
        if k not in keys:
            keys.append(k)
        zone.append(keys.index(k))
    assert o["zones"] == keys
    assert o["zone"] == zone
    assert len(keys) == 4 and zone[4] == ZONE_NONE and zone[5] == zone[0] != zone[2]


def test_zone_limit(packed):
    assert packed["packs_64"] == 64
    assert packed["packs_65"] == -1


def test_classes_and_counts(packed):
    o = packed
    N = len(o["nodes"])
    cls, counts = o["spread_class"], o["counts"]
    idents = []
    for p, pod in enumerate(o["pods"]):
        sels = _selectors(o, pod)
        ident = (pod["ns"], frozenset(i for i, _ in sels)) if sels else None
        idents.append(ident)
        if ident is None:
            assert cls[p] == SPREAD_NONE, p
            continue
        row = counts[cls[p] * N:(cls[p] + 1) * N]
        assert row == [_count(pod, sels, nd) for nd in o["nodes"]], p
    for p in range(len(cls)):
        for q in range(len(cls)):
            if idents[p] is not None and idents[q] is not None:
                assert (cls[p] == cls[q]) == (idents[p] == idents[q]), (p, q)
    assert len(counts) == N * (max(c for c in cls if c != SPREAD_NONE) + 1)


def test_the_named_cases(packed):
    """The cases the fixture was built for, spelled out."""
    o = packed
    N = len(o["nodes"])
    cls, counts = o["spread_class"], o["counts"]
    row = lambda p: counts[cls[p] * N:(cls[p] + 1) * N]   # noqa: E731
    # p0 and p7: the same labels in another order share a class; svc-web AND rs-fe (tier In fe, be); the terminating
    # web pod on node 1 and the web pod of namespace "other" on node 0 do not count
    assert cls[0] == cls[7]
    assert row(0) == [1, 1, 0, 1, 0, 2]
    # p1: only svc-web (rs-fe needs a tier label)
    assert row(1) == [1, 1, 0, 1, 0, 3]
    # p2: rc-db AND ss-db (tier DoesNotExist, app In db): the db pod with a tier on node 3 does not count; rc-empty
    # (an empty RC selector) selects nothing, else p3 and p8 would have a class
    assert row(2) == [0, 0, 1, 1, 0, 0]
    # p3 (no labels) and p8 (nothing selects it): no class
    assert cls[3] == SPREAD_NONE and cls[8] == SPREAD_NONE
    # p4: no labels, but svc-all's empty selector in "other" selects it and counts every live pod there
    assert row(4) == [1, 0, 1, 0, 1, 0]
    # p5: svc-all AND ss-web
    assert row(5) == [1, 0, 0, 0, 1, 0]
    # p6: svc-batch AND rs-notin (app NotIn db, web; role Exists); the invalid RS / StatefulSet selectors are skipped
    assert row(6) == [1, 1, 1, 0, 0, 0]
