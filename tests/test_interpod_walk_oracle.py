"""CPU: the walks under the MatchInterPodAffinity filter, restated twice.  tests/interpod_walk_ref.c decides each
(pod, node) on the packed columns (pyref_interpod_filter.pack plus pyref_interpod_walk.placed), looping over the bound
and the assumed pods; pyref_interpod_walk.walk decides it from the objects with the assumed pods appended to the existing
ones.  Both drive the oracle's first-fit walk and must agree, on the hand-built cases (whose placements are written
out) and on seeded random clusters."""

import numpy as np
import pytest

import interpod_filter_ref as fr
import interpod_walk_cases as cases
import interpod_walk_ref as iwr
import pyref_interpod_filter as pyf
import pyref_interpod_walk as pyw
from pyref_interpod_filter import Pod, Term


def _both(nodes, existing, pending, queue=None):
    snap = cases.snapshot(len(nodes), len(pending))
    cols = pyf.pack(nodes, existing, pending)
    placed = pyw.placed(nodes, existing, pending)
    obj = pyw.walk(snap, nodes, existing, pending, queue)
    col = iwr.replay(snap, cols, placed, queue)
    for k, name in enumerate(("prefilter", "node", "ready")):
        np.testing.assert_array_equal(col[k], obj[k], err_msg=name)
    for f in ("requested", "pod_count", "req_present"):
        np.testing.assert_array_equal(getattr(col[3].nodes, f), getattr(obj[3].nodes, f), err_msg=f)
    for f in ("matched", "flags"):
        np.testing.assert_array_equal(getattr(col[3].groups, f), getattr(obj[3].groups, f), err_msg=f)
    return col, cols, placed


@pytest.mark.parametrize("case", cases.CASES, ids=[c[0] for c in cases.CASES])
def test_cases(oracle, case):
    name, nodes, existing, pending, queue, want = case
    (_, node, ready, *_), _, _ = _both(nodes, existing, pending, cases.queue_of(case))
    assert node.tolist() == want
    if name == "eight-anti-workers":
        assert not ready.any()   # MinMember 8, five placed


def test_placed_agrees_with_filter_classes(oracle):
    # every placed match entry on a term some bound pod owns is an EXISTING entry of the pod's filter class: the
    # walk's first step then sees the round's verdicts
    for _, nodes, existing, pending, _, _ in cases.CASES + [_random_cluster(s) for s in range(8)]:
        (_, _, _, _, bcls, (boff, bterm, bown, _)), (pcls, (poff, pterm, prole, _)) = pyf.pack(nodes, existing, pending)
        owned = {int(bterm[k]) for c in bcls if c != pyf.IPF_NONE for k in range(boff[c], boff[c + 1]) if bown[k]}
        qcls, (qoff, qterm, qown, qmatch) = pyw.placed(nodes, existing, pending)
        for p in range(len(pending)):
            if qcls[p] == pyf.IPF_NONE:
                continue
            matched = {int(qterm[k]) for k in range(qoff[qcls[p]], qoff[qcls[p] + 1]) if qmatch[k]} & owned
            fc = pcls[p]
            existing_terms = set() if fc == pyf.IPF_NONE else \
                {int(pterm[k]) for k in range(poff[fc], poff[fc + 1]) if prole[k] == pyf.EXISTING}
            assert matched <= existing_terms


def _random_cluster(seed, n_nodes=7, n_existing=6, n_pending=10):
    rng = np.random.default_rng(seed)
    zones = [None, "a", "b", "c"]
    nodes = {}
    for i in range(n_nodes):
        lab = {cases.H: f"n{i}"}
        z = zones[rng.integers(0, len(zones))]
        if z is not None:
            lab[cases.Z] = z
        nodes[f"n{i}"] = lab
    apps, keys, nss = ["x", "y", "z"], [cases.H, cases.Z, cases.Z, ""], ["default", "default", "other"]

    def term():
        sel = {"app": apps[rng.integers(0, len(apps))]} if rng.random() < 0.9 else {}
        return Term(sel, keys[rng.integers(0, len(keys))], [nss[rng.integers(0, 2)]] if rng.random() < 0.2 else [])

    def pod(name, node=None):
        return Pod(name, nss[rng.integers(0, len(nss))], {"app": apps[rng.integers(0, len(apps))]}, node=node,
                   affinity=[term() for _ in range(int(rng.random() < 0.3) * int(rng.integers(1, 3)))],
                   anti=[term() for _ in range(int(rng.random() < 0.4))])

    existing = [pod(f"e{i}", f"n{rng.integers(0, n_nodes)}") for i in range(n_existing)]
    pending = [pod(f"p{i}") for i in range(n_pending)]
    queue = rng.permutation(n_pending).astype(np.uint32)
    return f"random-{seed}", nodes, existing, pending, queue, None


@pytest.mark.parametrize("seed", range(24))
def test_random_clusters(oracle, seed):
    _, nodes, existing, pending, queue, _ = _random_cluster(seed)
    col, cols, placed = _both(nodes, existing, pending, queue)
    # the first step sees the round's verdicts
    p0 = int(queue[0])
    v = fr.verdicts(cols, len(nodes), [p0])[0]
    first = iwr.replay(cases.snapshot(len(nodes), len(pending)), cols, placed, queue[:1])[1][0]
    passing = np.flatnonzero(v == fr.PASS)
    assert first == (passing[0] if len(passing) else -1)
