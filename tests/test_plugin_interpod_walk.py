"""BatchSchedulingPlugin and the MatchInterPodAffinity filter in its walks (tests/cpp/plugin_interpod_walk_test.cpp).

CPU: PackInterPodFilter's placed classes say, for every ordered pair of pending pods, what the object restatement
(tests/pyref_interpod_filter.py) says one pod's placement does to the other: which topology keys its anti-affinity
blocks for the other (step 1), which keys it counts in for the other's anti-affinity (step 4) and affinity set
(step 3); a pod's match entries on the bound pods' terms are its EXISTING entries; and packing without the placed side
leaves every other column as it was.  GPU: with SetInterPodAffinityFilter(true) ReplayQueue refuses to run until
SetInterPodAffinityFilterInWalks(true); then its first-fit walk equals the object walk (each pod on the first node that
passes against the bound pods and the pods placed before it), its priority walk places a pod exactly when some node
passes and only on such a node, and UpdateNodes repacks the placed side with the rest."""
import json
import subprocess

import pytest

import native
import pyref_interpod_filter as py

NONE = py.IPF_NONE
BASE = ("keys", "n_values", "topo", "term_key", "bound_node", "bound_class", "bound_classes", "pod_class", "pod_classes")


def _run(*args):
    return json.loads(subprocess.check_output([native.cpp_program("plugin_interpod_walk_test"), *args], text=True))


@pytest.fixture(scope="module")
def out():
    return _run()


def _term(t):
    sel = t["selector"]
    return py.Term(py.INVALID if sel == "invalid" else sel, t["key"], list(t["namespaces"]))


def _pod(o, node=None):
    return py.Pod(o["name"], o["ns"], dict(o["labels"]), node, [_term(t) for t in o["affinity"]],
                  [_term(t) for t in o["anti"]], o["terminating"])


def _objects(sc):
    nodes = {n["name"]: (dict(n["labels"]) if n["has_node"] else {}) for n in sc["nodes"]}
    existing = [_pod(b, n["name"]) for n in sc["nodes"] if n["has_node"] for b in n["pods"]]
    return nodes, existing, [_pod(p) for p in sc["pods"]]


def _entries(offset, cls, *cols):
    """{term: (col values...)} of class cls (none: {})."""
    if cls == NONE:
        return {}
    return {cols[0][k]: tuple(c[k] for c in cols[1:]) for k in range(offset[cls], offset[cls + 1])}


def test_plain_columns_are_unchanged(out):
    for sc in out["scenarios"]:
        for f in BASE:
            assert sc["plain"][f] == sc["packed"][f], f
        assert sc["plain"]["placed_class"] == [] and sc["plain"]["placed_classes"] == [[0], [], [], []]
        assert len(sc["packed"]["placed_class"]) == len(sc["pods"])


@pytest.mark.parametrize("scenario", range(3))
def test_placed_classes_against_objects(out, scenario):
    sc = out["scenarios"][scenario]
    k = sc["packed"]
    _, _, pending = _objects(sc)
    key = [k["keys"][i] for i in k["term_key"]]
    poff, pterm, prole, _ = k["pod_classes"]
    qoff, qterm, qown, qmatch = k["placed_classes"]
    boff, bterm, bown, _ = k["bound_classes"]
    owned = {bterm[j] for j in range(len(bterm)) if bown[j]}
    filt = [_entries(poff, c, pterm, prole) for c in k["pod_class"]]
    placed = [_entries(qoff, c, qterm, qown, qmatch) for c in k["placed_class"]]
    for p, pp in enumerate(pending):
        own = {t for t, (o, _) in placed[p].items() if o}
        assert own == {t for t, (r,) in filt[p].items() if r == py.ANTI}
        match = {t for t, (_, m) in placed[p].items() if m}
        assert match & owned == {t for t, (r,) in filt[p].items() if r == py.EXISTING}
        assert all(o or m for o, m in placed[p].values())
        for q, qq in enumerate(pending):
            # step 1: the keys on which p, once placed, keeps q out
            got = {key[t] for t in own if placed[q].get(t, (0, 0))[1]}
            assert got == {u.key for u in pp.anti if py.pod_matches_term(qq, u, pp.ns)}, (p, q)
            # step 4: the keys on which p counts against q's anti-affinity
            got = {key[t] for t, (r,) in filt[q].items() if r == py.ANTI and t in match}
            assert got == {u.key for u in qq.anti if py.pod_matches_term(pp, u, qq.ns)}, (p, q)
            # step 3: the keys on which p counts for q's affinity set (it matches the whole set)
            got = {key[t] for t, (r,) in filt[q].items() if r == py.AFFINITY and t in match}
            whole = bool(qq.affinity) and all(py.pod_matches_term(pp, x, qq.ns) for x in qq.affinity)
            assert got == ({x.key for x in qq.affinity} if whole else set()), (p, q)


def test_scenarios_cover_the_relations(out):
    n_e = n_n = n_a = 0
    for sc in out["scenarios"]:
        _, _, pending = _objects(sc)
        for pp in pending:
            for qq in pending:
                n_e += any(py.pod_matches_term(qq, u, pp.ns) for u in pp.anti)
                n_n += any(py.pod_matches_term(pp, u, qq.ns) for u in qq.anti)
                n_a += bool(qq.affinity) and all(py.pod_matches_term(pp, x, qq.ns) for x in qq.affinity)
    assert n_e and n_n and n_a


def _object_walk(sc, placements=None):
    """The first-fit walk from objects in the plugin's queue order, or (placements given) the check of another walk's
    placements: each placed pod passes its node and a pod is left out only when no node passes."""
    nodes, existing, pending = _objects(sc)
    names = [n["name"] for n in sc["nodes"] if n["has_node"]]
    index = {n["name"]: i for i, n in enumerate(sc["nodes"])}
    assumed, got = [], []
    for pos, p in enumerate(sc["queue"]):
        pod = pending[p]
        ok = [n for n in names if py.verdict(pod, n, nodes, existing + assumed) is None]
        if placements is None:
            n = index[ok[0]] if ok else -1
        else:
            n = placements[pos]
            assert (n >= 0) == bool(ok), pos
            assert n < 0 or sc["nodes"][n]["name"] in ok, pos
        got.append(n)
        if n >= 0:
            assumed.append(py.Pod(pod.name, pod.ns, pod.labels, sc["nodes"][n]["name"], pod.affinity, pod.anti))
    return got


@pytest.mark.gpu
def test_plugin_walks(pkg):
    o = _run("gpu")
    placed_any = False
    for sc in o["scenarios"]:
        assert sc["refused_without_opt_in"]
        assert sc["first_fit"] == _object_walk(sc)
        _object_walk(sc, sc["priority"])
        assert sc["first_fit_after_update_nodes"] == sc["first_fit"]
        placed_any |= any(n >= 0 for n in sc["first_fit"]) and any(n < 0 for n in sc["first_fit"])
    assert placed_any
