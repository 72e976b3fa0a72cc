"""CPU: the two restatements of the InterPodAffinity priority (tests/interpod_priority_ref.c over packed columns, and
tests/pyref_interpod_priority.py over objects) agree on random objects, alone and with the resource weights and the
ratio term; on the binary64 pins of the reduce; on both extremes starting at 0; on a non-fitting node with the extreme
raw; on nodes without the key; on terminating bound pods, nil and empty selectors, empty and listed namespaces, the
hard weight at 0, 1 and 100, and a pod scored only through bound pods' terms.  With weight 0 the lists are the
existing ones."""
import numpy as np
import pytest

import interpod_cases as ic
import interpod_priority_ref as ir
import node_priority_ref as npr
import priority_ref as pr
import pyref_interpod_priority as pyi
import ratio_priority_ref as rr
from oracle import oracle
from randsnap import S, random_snapshot

HOST, ZONE = ic.HOST, ic.ZONE


def _agree(snap, nz, K, objs, w, hard=1, ratio=npr.NO_RATIO, weights=(1, 0, 1)):
    pending, bound, labels = objs
    cols = ic.columns(pending, bound, labels, hard)
    nodes, scores = ir.priority_rows(snap, nz[0], nz[1], K, cols, w, ratio, weights)
    want = pyi.priority_rows(snap, nz[0], nz[1], K, pending, bound, labels, w, hard, ratio, weights)
    for p, row in enumerate(want):
        assert nodes[p].tolist() == [n for n, _ in row], p
        assert scores[p].tolist() == [s for _, s in row], p
    return nodes, scores


def _fit(snap):
    """[P, N] bool: the fit set of every pod (the oracle's fit bitmap)."""
    bm = oracle.round(snap, want_bitmap=True).fit_bitmap
    bits = np.unpackbits(bm.view(np.uint8), axis=1, bitorder="little")[:, :snap.nodes.n]
    return bits.astype(bool)


def _raw(objs, p, hard=1):
    pending, bound, labels = objs
    return ir.raw_matrix(ic.columns(pending, bound, labels, hard), len(labels), [p])[0]


def test_binary64_pins():
    # raws {-7, 22, 43}: min -7, max 43; 100 * (29 / 50) = 57.99999999999999 in binary64
    assert [ir.ipa_score(r, -7, 43) for r in (-7, 22, 43)] == [0, 57, 100]
    assert pyi.reduce({0: -7, 1: 22, 2: 43}) == {0: 0, 1: 57, 2: 100}
    # both extremes start at 0: all positive, all negative, all zero
    assert pyi.reduce({0: 10, 1: 20}) == {0: 50, 1: 100}
    assert [ir.ipa_score(r, 0, 20) for r in (10, 20)] == [50, 100]
    assert pyi.reduce({0: -10, 1: -20}) == {0: 50, 1: 0}
    assert [ir.ipa_score(r, -20, 0) for r in (-10, -20)] == [50, 0]
    assert pyi.reduce({0: 0, 1: 0}) == {0: 0, 1: 0} and ir.ipa_score(0, 0, 0) == 0
    # the widest raws the caps allow convert exactly
    assert ir.ipa_score(1 << 47, -(1 << 47), 1 << 47) == 100 and ir.ipa_score(0, -(1 << 47), 1 << 47) == 50


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("w", [1, 3])
def test_random_objects_agree(seed, w):
    snap = random_snapshot(3000 + seed, P=40, N=30, G=6, L=5 + seed % 3)
    nz = S.nonzero_requests(snap, seed)
    objs = ic.random_objects(seed, snap.nodes.n, snap.pods.n)
    _agree(snap, nz, 7, objs, w)


@pytest.mark.parametrize("seed", range(2))
@pytest.mark.parametrize("weights", [(1, 0, 1), (2, 3, 5)])
@pytest.mark.parametrize("ratio_on", [False, True])
def test_combined_with_resource_weights_and_ratio(seed, weights, ratio_on):
    snap = random_snapshot(3050 + seed, P=30, N=25, G=6, L=6)
    nz = S.nonzero_requests(snap, seed)
    ratio = (3, rr.BIN_PACK, [1, 1, 0, 0, 2, 1]) if ratio_on else npr.NO_RATIO
    _agree(snap, nz, 9, ic.random_objects(seed + 7, snap.nodes.n, snap.pods.n), 2, 1, ratio, weights)


@pytest.mark.parametrize("hard", [0, 1, 100])
def test_hard_weight(hard):
    snap = random_snapshot(3060, P=30, N=25, G=6)
    nz = S.nonzero_requests(snap, 1)
    _agree(snap, nz, 8, ic.random_objects(11, snap.nodes.n, snap.pods.n), 1, hard)


def test_hard_weight_scales_required_terms_only():
    labels = [{HOST: "n0", ZONE: "z"}, {HOST: "n1", ZONE: "z"}, {HOST: "n2"}]
    e = pyi.PodObj("a", {"app": "db"}, node=0, required=[pyi.Term(pyi.Selector({"app": "web"}), (), ZONE)])
    p = pyi.PodObj("a", {"app": "web"})
    objs = ([p], [e], labels)
    for hard, want in ((0, [0, 0, 0]), (1, [1, 1, 0]), (100, [100, 100, 0])):
        assert list(pyi.raw_scores(p, [e], labels, hard).values()) == want
        assert _raw(objs, 0, hard).tolist() == want


def test_zero_weight_gives_existing_lists():
    snap = random_snapshot(3070, P=40, N=30, G=6)
    nz = S.nonzero_requests(snap, 2)
    nodes, scores = _agree(snap, nz, 8, ic.random_objects(3, snap.nodes.n, snap.pods.n), 0)
    n0, s0 = pr.priority_rows(snap, nz[0], nz[1], 8)
    assert np.array_equal(nodes, n0) and np.array_equal(scores, s0)


def test_non_fitting_node_with_the_extreme_raw_moves_nothing():
    snap = random_snapshot(3080, P=40, N=30, G=6)
    nz = S.nonzero_requests(snap, 5)
    fit = _fit(snap)
    n_out = next(n for n in range(snap.nodes.n) if not fit[:, n].all())
    pods = np.nonzero(~fit[:, n_out] & fit.any(axis=1))[0]
    assert len(pods)
    pending, bound, labels = ic.random_objects(5, snap.nodes.n, snap.pods.n)
    base = _agree(snap, nz, 30, (pending, bound, labels), 1)
    # heavy bound pods on n_out, in a namespace no pending pod's term names, attracting every pending pod to n_out's
    # hostname value alone: n_out gets the largest raw of every pod
    term = pyi.Term(pyi.Selector(), ic.NAMESPACES, HOST)
    heavy = [pyi.PodObj("z", {"app": "x"}, node=n_out, preferred=[(100, term)]) for _ in range(5)]
    more = _agree(snap, nz, 30, (pending, bound + heavy, labels), 1)
    assert np.array_equal(base[0][pods], more[0][pods]) and np.array_equal(base[1][pods], more[1][pods])


def test_nodes_without_the_key():
    labels = [{HOST: "n0", ZONE: "z"}, {HOST: "n1"}, {HOST: "n2", ZONE: "z"}]
    e = pyi.PodObj("a", {"app": "db"}, node=1)   # its node has no zone: no zone term reaches any node
    p = pyi.PodObj("a", {"app": "web"}, preferred=[(7, pyi.Term(pyi.Selector({"app": "db"}), (), ZONE))])
    assert list(pyi.raw_scores(p, [e], labels).values()) == [0, 0, 0]
    assert _raw(([p], [e], labels), 0).tolist() == [0, 0, 0]
    e.node = 0
    assert list(pyi.raw_scores(p, [e], labels).values()) == [7, 0, 7]
    assert _raw(([p], [e], labels), 0).tolist() == [7, 0, 7]


def test_terminating_bound_pods_count():
    labels = [{HOST: "n0"}, {HOST: "n1"}]
    e = pyi.PodObj("a", {"app": "db"}, node=1, terminating=True)
    p = pyi.PodObj("a", {"app": "web"}, anti=[(9, pyi.Term(pyi.Selector({"app": "db"}), (), HOST))])
    assert list(pyi.raw_scores(p, [e], labels).values()) == [0, -9]
    assert _raw(([p], [e], labels), 0).tolist() == [0, -9]


def test_nil_and_empty_selectors():
    labels = [{HOST: "n0"}, {HOST: "n1"}]
    e = pyi.PodObj("a", {"app": "db"}, node=0)
    for sel, want in ((None, [0, 0]), (pyi.Selector(), [5, 0])):
        p = pyi.PodObj("a", {"app": "web"}, preferred=[(5, pyi.Term(sel, (), HOST))])
        assert list(pyi.raw_scores(p, [e], labels).values()) == want
        assert _raw(([p], [e], labels), 0).tolist() == want


def test_namespaces_empty_and_listed():
    labels = [{HOST: "n0"}, {HOST: "n1"}]
    e = pyi.PodObj("b", {"app": "db"}, node=1)
    sel = pyi.Selector({"app": "db"})
    for ns, want in (((), [0, 0]), (("b",), [0, 4]), (("a", "c"), [0, 0]), (("c", "b"), [0, 4])):
        p = pyi.PodObj("a", {"app": "web"}, preferred=[(4, pyi.Term(sel, ns, HOST))])
        assert list(pyi.raw_scores(p, [e], labels).values()) == want
        assert _raw(([p], [e], labels), 0).tolist() == want
    # a bound pod's empty namespaces mean its own namespace, not the pending pod's
    e2 = pyi.PodObj("b", {"app": "db"}, node=0, preferred=[(6, pyi.Term(pyi.Selector({"app": "web"}), (), HOST))])
    for ns, want in (("a", [0, 0]), ("b", [6, 0])):
        p = pyi.PodObj(ns, {"app": "web"})
        assert list(pyi.raw_scores(p, [e2], labels).values()) == want
        assert _raw(([p], [e2], labels), 0).tolist() == want


def test_pod_matched_only_through_bound_pods_terms():
    """A pod without terms of its own scores through the bound pods' affinity (+) and anti-affinity (-)."""
    snap = random_snapshot(3090, P=30, N=25, G=6)
    nz = S.nonzero_requests(snap, 6)
    pending, bound, labels = ic.random_objects(9, snap.nodes.n, snap.pods.n, per_node=4)
    for p in pending:
        p.required, p.preferred, p.anti = [], [], []
    raws = ir.raw_matrix(ic.columns(pending, bound, labels), snap.nodes.n)
    assert (raws > 0).any() and (raws < 0).any()
    _agree(snap, nz, 10, (pending, bound, labels), 1)


def test_invalid_selectors_give_no_class():
    snap = random_snapshot(3095, P=30, N=25, G=6)
    nz = S.nonzero_requests(snap, 7)
    pending, bound, labels = ic.random_objects(12, snap.nodes.n, snap.pods.n)
    bad = pyi.Term(pyi.Selector({}, [("tier", "Exists", ["x"])]), (), HOST)
    pending[3].preferred.append((5, bad))   # its own invalid term: only this pod scores 0
    pk = pyi.pack(pending, bound, labels)
    assert pk["pods"][0][3] == pyi.IPA_NONE
    _agree(snap, nz, 8, (pending, bound, labels), 1)
    bound[0].anti.append((5, bad))   # a bound pod's: every pending pod
    pk = pyi.pack(pending, bound, labels)
    assert set(pk["pods"][0]) == {pyi.IPA_NONE}
    _agree(snap, nz, 8, (pending, bound, labels), 1)


def test_pods_without_fitting_nodes():
    snap = random_snapshot(3099, P=30, N=25, G=6)
    snap.pods.req[0, :10] = 1 << 55   # no node has that much cpu left
    nz = S.nonzero_requests(snap, 8)
    nodes, scores = _agree(snap, nz, 5, ic.random_objects(13, snap.nodes.n, snap.pods.n), 1)
    assert (nodes[:10] == -1).all() and (scores[:10] == np.iinfo(np.int64).min).all()


def test_generated_columns_within_caps():
    snap = random_snapshot(3100, P=50, N=40, G=6)
    (nv, topo, tkey, bnode, bcls, bcl), (pcls, pcl) = S.node_interpod(snap, 1)
    for off, term, own, match in (bcl, pcl):
        assert off[0] == 0 and (np.diff(off) <= 64).all() and (np.abs(own) <= 1 << 16).all() and set(match) <= {0, 1}
        for c in range(len(off) - 1):
            assert len(set(term[off[c]:off[c + 1]])) == off[c + 1] - off[c]
    assert (pcls == S.IPA_NONE).any() and (bcls == S.IPA_NONE).any()
    raws = ir.raw_matrix(S.node_interpod(snap, 1), snap.nodes.n)
    assert (raws > 0).any() and (raws < 0).any()
