"""CPU: the two restatements of the MatchInterPodAffinity filter agree — tests/pyref_interpod_filter.py from objects
(upstream's topology-pair maps) and tests/interpod_filter_ref.c over the packed columns (a loop over the bound pods) —
on the hand-built cases with their written answers and on random objects; the message entries and their order; the
seeded generator's columns."""
from importlib import import_module

import numpy as np
import pytest

import interpod_filter_cases as cases
import interpod_filter_ref as fr
import pyref_interpod_filter as py
from randsnap import S, random_snapshot

_CODE = {"": fr.PASS, "E": fr.FAIL_E, "A": fr.FAIL_A, "N": fr.FAIL_N}


@pytest.mark.parametrize("case", cases.CASES, ids=[c[0] for c in cases.CASES])
def test_cases(case):
    _, nodes, existing, pending, answers = case
    names = list(nodes)
    for p in pending:
        got = [py.verdict(p, n, nodes, existing) or "" for n in names]
        assert got == answers[p.name], p.name
    v = fr.verdicts(py.pack(nodes, existing, pending), len(names))
    for k, p in enumerate(pending):
        assert v[k].tolist() == [_CODE[x] for x in answers[p.name]], p.name


def _random_objects(rng, n_nodes=12, n_existing=30, n_pending=25):
    zones = ["a", "b", "c", None]
    nodes = {}
    for i in range(n_nodes):
        lab = {py_key: f"n{i}" for py_key in ["kubernetes.io/hostname"]}
        z = zones[int(rng.integers(0, 4))]
        if z is not None:
            lab["zone"] = z
        if rng.random() < 0.5:
            lab["rack"] = f"r{i // 3}"
        nodes[f"n{i}"] = lab
    keys = ["kubernetes.io/hostname", "zone", "rack", ""]
    apps, nss = ["x", "y", "z"], ["default", "other"]

    def selector():
        r = rng.random()
        if r < 0.05:
            return None
        if r < 0.1:
            return {}
        if r < 0.13:
            return py.INVALID
        sel = {"app": apps[int(rng.integers(0, 3))]}
        if rng.random() < 0.3:
            sel["tier"] = str(int(rng.integers(0, 2)))
        return sel

    def terms(k):
        return [py.Term(selector(), keys[int(rng.integers(0, 4))],
                        [] if rng.random() < 0.7 else [nss[int(rng.integers(0, 2))]]) for _ in range(k)]

    def pod(name, node=None):
        labels = {"app": apps[int(rng.integers(0, 3))], "tier": str(int(rng.integers(0, 2)))}
        return py.Pod(name, nss[int(rng.integers(0, 2))], labels, node,
                      terms(int(rng.integers(0, 3)) if rng.random() < 0.5 else 0),
                      terms(int(rng.integers(0, 3)) if rng.random() < 0.5 else 0))

    names = list(nodes) + ["gone"]   # a pod on a node outside the snapshot contributes nothing
    existing = [pod(f"e{i}", names[int(rng.integers(0, len(names)))]) for i in range(n_existing)]
    pending = [pod(f"p{i}") for i in range(n_pending)]
    return nodes, existing, pending


@pytest.mark.parametrize("seed", range(12))
def test_restatements_agree(seed):
    nodes, existing, pending = _random_objects(np.random.default_rng(seed))
    names = list(nodes)
    v = fr.verdicts(py.pack(nodes, existing, pending), len(names))
    want = np.array([[_CODE[py.verdict(p, n, nodes, existing) or ""] for n in names] for p in pending], np.uint8)
    np.testing.assert_array_equal(v, want)
    assert (v != fr.PASS).any() and (v == fr.PASS).any()


def test_message():
    eng = import_module("batch-scheduler_b200.engine")
    row, ip, n = cases.MESSAGE_ROW
    assert eng.format_fit_error(row, 4, n, interpod=ip) == cases.MESSAGE
    # without a companion, and with an all-zero one, the message is bs_format_fit_error's
    plain = eng.format_fit_error(row, 4, n)
    assert plain == "0/6 nodes are available: 2 Insufficient cpu."
    assert eng.format_fit_error(row, 4, n, interpod=(0, 0, 0)) == plain
    assert eng.format_fit_error([0] * 8, 4, 3, interpod=(0, 0, 3)) == (
        "0/3 nodes are available: 3 node(s) didn't match pod affinity/anti-affinity, "
        "3 node(s) didn't match pod anti-affinity rules.")


def test_generator():
    snap = random_snapshot(77, P=300, N=200, G=40, L=5, case="mixed")
    cols = S.node_interpod_filter(snap, 5)
    again = S.node_interpod_filter(snap, 5)
    for a, b in zip(np.concatenate([np.ravel(x) for x in cols[0][:5]]), np.concatenate([np.ravel(x) for x in again[0][:5]])):
        assert a == b
    v = fr.verdicts(cols, snap.nodes.n)
    assert set(np.unique(v).tolist()) == {fr.PASS, fr.FAIL_E, fr.FAIL_A, fr.FAIL_N}
    # the roles the generator promises: hostname anti-affinity, zone affinity, bound pods' anti-affinity
    roles = set(cols[1][1][2].tolist())
    assert roles == {py.AFFINITY, py.ANTI, py.EXISTING}
