"""GPU: every refusal of the priority and filter side tables, table-driven.  Each side upload (the non-zero columns,
the TaintToleration / NodeAffinity preferences, locality, SelectorSpread, InterPodAffinity and the
MatchInterPodAffinity filter, node and pod halves) is called through the C ABI with one wrong input at a time, and
the test pins the return code, the exact bs_last_error text and that the side is gone afterwards: the next round,
with every weight on, answers BS_E_STATE with that side's message.  The evaluation checks of bs_evaluate and the
non-zero and locality checks of bs_replay_priority are pinned the same way (code and text)."""
import ctypes as C
import importlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

S = importlib.import_module("batch-scheduler_b200.snapshot")
capi = importlib.import_module("batch-scheduler_b200.capi")

OK, INVAL, RANGE, STATE, INDEX = capi.BS_OK, capi.BS_E_INVAL, capi.BS_E_RANGE, capi.BS_E_STATE, capi.BS_E_INDEX
L = 4

# what bs_evaluate answers once a side is gone (every other side present, every weight on)
TABLES = "bs_evaluate: upload nodes, groups and pods first"
NZ = "bs_evaluate: BS_OUT_PRIORITY needs the node and pod non-zero columns"
PREF = "bs_evaluate: a non-zero node priority weight needs the node and pod preference columns"
LOC = "bs_evaluate: a non-zero ImageLocality weight needs the node and pod image columns"
SPREAD = "bs_evaluate: a non-zero SelectorSpread weight needs the node and pod spread columns"
IPA = "bs_evaluate: a non-zero InterPodAffinity weight needs the node and pod inter-pod sides"
IPF = "bs_evaluate: the MatchInterPodAffinity filter needs its node and pod sides"


def a32(*v):
    return np.array(v, np.uint32)


_ALIVE = []   # every array handed to the C ABI in a test stays alive until its end


def ptr(a):
    if a is None:
        return None
    a = np.ascontiguousarray(a)
    _ALIVE.append(a)
    return capi.ptr(a)


# ---- valid sides of an N-node, P-pod engine ---------------------------------------------------------------------
def ipa_node(N, nv=(1,), topo=None, tkey=(0,), bnode=(), bcls=(), cl=((0,), (), (), ()), null=(), **over):
    """A bs_interpod_nodes struct and the arrays it points at; `over` replaces counts, `null` names NULL columns."""
    nv = np.array(nv, np.uint32)
    topo = np.zeros((len(nv), N), np.uint32) if topo is None else np.array(topo, np.uint32)
    arr = dict(n_values=nv, topo=topo, term_key=np.array(tkey, np.uint32), bound_node=np.array(bnode, np.uint32),
               bound_class=np.array(bcls, np.uint32), class_offset=np.array(cl[0], np.uint32),
               term=np.array(cl[1], np.uint32), own=np.array(cl[2], np.int32), match=np.array(cl[3], np.uint8))
    cnt = dict(n_nodes=N, n_keys=len(nv), n_terms=len(arr["term_key"]), n_bound=len(arr["bound_node"]),
               n_classes=max(len(arr["class_offset"]) - 1, 0))
    cnt.update(over)
    p = {k: None if k in null else ptr(v) for k, v in arr.items()}
    cls = capi.InterpodClassesC(cnt["n_classes"], p["class_offset"], p["term"], p["own"], p["match"])
    t = capi.InterpodNodesC(cnt["n_nodes"], cnt["n_keys"], p["n_values"], p["topo"], cnt["n_terms"], p["term_key"],
                            cnt["n_bound"], p["bound_node"], p["bound_class"], cls)
    return t, arr


def ipa_pods(P, pcls=None, cl=((0, 1), (0,), (1,), (1,)), null=(), **over):
    arr = dict(pod_class=np.full(P, capi.IPA_NONE, np.uint32) if pcls is None else np.array(pcls, np.uint32),
               class_offset=np.array(cl[0], np.uint32), term=np.array(cl[1], np.uint32),
               own=np.array(cl[2], np.int32), match=np.array(cl[3], np.uint8))
    cnt = dict(n_pods=P, n_classes=max(len(arr["class_offset"]) - 1, 0))
    cnt.update(over)
    p = {k: None if k in null else ptr(v) for k, v in arr.items()}
    cls = capi.InterpodClassesC(cnt["n_classes"], p["class_offset"], p["term"], p["own"], p["match"])
    return capi.InterpodPodsC(cnt["n_pods"], p["pod_class"], cls), arr


def ipf_pods(P, pcls=None, off=(0, 1), term=(0,), role=(0,), self_match=(0,), null=(), **over):
    arr = dict(pod_class=np.full(P, capi.IPF_NONE, np.uint32) if pcls is None else np.array(pcls, np.uint32),
               class_offset=np.array(off, np.uint32), term=np.array(term, np.uint32), role=np.array(role, np.uint8),
               self_match=np.array(self_match, np.uint8))
    cnt = dict(n_pods=P, n_classes=max(len(arr["class_offset"]) - 1, 0))
    cnt.update(over)
    p = {k: None if k in null else ptr(v) for k, v in arr.items()}
    return capi.InterpodFilterPodsC(cnt["n_pods"], p["pod_class"], cnt["n_classes"], p["class_offset"], p["term"],
                                    p["role"], p["self_match"]), arr


def node_sides(eng, N):
    lib, h = eng.lib, eng.h
    z64, w = np.zeros(2 * N, np.int64), np.zeros(N, np.int32)
    words = (N + 31) // 32
    assert lib.bs_upload_node_nonzero(h, N, ptr(z64)) == OK
    assert lib.bs_upload_node_preferences(h, N, ptr(np.zeros(N, np.uint64)), 1, ptr(w)) == OK
    assert lib.bs_upload_node_locality(h, N, 1, ptr(np.array([1 << 20], np.int64)), ptr(np.zeros(words, np.uint32)),
                                       ptr(np.zeros(N, np.uint64))) == OK
    assert lib.bs_upload_node_spread(h, N, 1, ptr(np.zeros(N, np.uint8)), 1, ptr(w)) == OK
    t, _ = ipa_node(N)
    assert lib.bs_upload_node_interpod(h, C.byref(t)) == OK
    t, _ = ipa_node(N)
    assert lib.bs_upload_node_interpod_filter(h, C.byref(t)) == OK


def pod_sides(eng, P):
    lib, h = eng.lib, eng.h
    assert lib.bs_upload_pod_nonzero(h, P, ptr(np.zeros(2 * P, np.int64))) == OK
    assert lib.bs_upload_pod_preferences(h, P, ptr(np.zeros(P, np.uint64)), ptr(np.zeros(P, np.uint32))) == OK
    assert lib.bs_upload_pod_locality(h, P, ptr(np.zeros(P, np.uint32)), 1, ptr(a32(0, 1)), ptr(a32(0)),
                                      ptr(np.zeros(P, np.uint8))) == OK
    assert lib.bs_upload_pod_spread(h, P, ptr(np.zeros(P, np.uint32))) == OK
    t, _ = ipa_pods(P)
    assert lib.bs_upload_pod_interpod(h, C.byref(t)) == OK
    t, _ = ipf_pods(P)
    assert lib.bs_upload_pod_interpod_filter(h, C.byref(t)) == OK


@pytest.fixture
def eng(pkg):
    """The README scenario (1 node, 10 pods) with every side uploaded, every weight on and one clean round."""
    snap = S.readme_scenario()
    e = pkg.Engine(L, 0, fit_bitmap=False, priority_k=4)
    e.upload(snap)
    e.snap = snap
    node_sides(e, snap.nodes.n)
    pod_sides(e, snap.pods.n)
    e.set_node_priority_weights(1, 1)
    e.set_locality_weights(1, 1)
    e.set_spread_weight(1)
    e.set_interpod_weight(1)
    e.set_interpod_filter(True)
    assert evaluate(e) == (OK, "")
    yield e
    e.close()
    _ALIVE.clear()


def last_error(eng):
    return eng.lib.bs_last_error(eng.h).decode()


def evaluate(eng):
    try:
        eng.evaluate()
    except capi.BsError as x:
        return x.code, last_error(eng)
    return OK, ""


def replay_priority(eng):
    try:
        eng.replay(priority=True, after_state=False)
    except capi.BsError as x:
        return x.code, last_error(eng)
    return OK, ""


def break_nodes(eng):
    """A node table that fails its range check: the engine is left without one."""
    nt = S.readme_scenario().nodes
    nt.alloc[0, 0] = 1 << 60
    with pytest.raises(capi.BsError):
        eng.upload_nodes(nt)


def break_pods(eng):
    pt = S.readme_scenario().pods
    pt.req[0, 0] = 1 << 60
    with pytest.raises(capi.BsError):
        eng.upload_pods(pt)


# ---- the uploads' refusals: (id, prepare, call(lib, h, N, P), code, text, bs_evaluate's message afterwards) -------
def _nz(half):
    fn, n, tab, first = (("bs_upload_node_nonzero", "n_nodes", "node", "nodes") if half == "node" else
                         ("bs_upload_pod_nonzero", "n_pods", "pod", "pods"))
    size = (lambda N, P: N) if half == "node" else (lambda N, P: P)
    brk = break_nodes if half == "node" else break_pods
    up = lambda lib, h, k, a: getattr(lib, fn)(h, k, ptr(a))   # noqa: E731
    return [
        (f"{fn}-state", brk, lambda lib, h, N, P: up(lib, h, size(N, P), np.zeros(2 * size(N, P), np.int64)),
         STATE, f"{fn}: upload {first} first", TABLES),
        (f"{fn}-size", None, lambda lib, h, N, P: up(lib, h, size(N, P) + 1, np.zeros(2 * size(N, P) + 2, np.int64)),
         INVAL, f"{fn}: {n} differs from the {tab} table's", NZ),
        (f"{fn}-null", None, lambda lib, h, N, P: up(lib, h, size(N, P), None), INVAL, f"{fn}: null column", NZ),
        (f"{fn}-range", None, lambda lib, h, N, P: up(lib, h, size(N, P), np.full(2 * size(N, P), -1, np.int64)),
         RANGE, "non-zero request outside [0, 2^56]", NZ),
    ]


def _pref_node(lib, h, N, n=None, taints=True, classes=1, weights=None, null_w=False):
    n = N if n is None else n
    w = np.zeros(max(classes * n, 1), np.int32) if weights is None else weights
    return lib.bs_upload_node_preferences(h, n, ptr(np.zeros(max(n, 1), np.uint64)) if taints else None, classes,
                                          None if null_w else ptr(w))


def _pref_pod(lib, h, P, n=None, null=False):
    n = P if n is None else n
    return lib.bs_upload_pod_preferences(h, n, ptr(np.zeros(max(n, 1), np.uint64)),
                                         None if null else ptr(np.zeros(max(n, 1), np.uint32)))


def _loc_node(lib, h, N, n=None, n_images=1, size=(1 << 20,), avoid=True):
    n = N if n is None else n
    words = max((n + 31) // 32, 1)
    return lib.bs_upload_node_locality(h, n, n_images, ptr(np.array(size, np.int64)),
                                       ptr(np.zeros(max(n_images, 1) * words if n_images < 1 << 20 else words,
                                                    np.uint32)),
                                       ptr(np.zeros(max(n, 1), np.uint64)) if avoid else None)


def _loc_pod(lib, h, P, n=None, n_classes=1, off=(0, 1), ids=(0,), cls=None, abit=None, avoid=True):
    n = P if n is None else n
    cls = np.zeros(max(n, 1), np.uint32) if cls is None else np.array(cls, np.uint32)
    abit = np.zeros(max(n, 1), np.uint8) if abit is None else np.array(abit, np.uint8)
    return lib.bs_upload_pod_locality(h, n, ptr(cls), n_classes, ptr(np.array(off, np.uint32)),
                                      ptr(np.array(ids, np.uint32)), ptr(abit) if avoid else None)


def _spread_node(lib, h, N, n=None, n_zones=1, zone=None, classes=1, counts=None, null_zone=False, null_counts=False):
    n = N if n is None else n
    zone = np.zeros(max(n, 1), np.uint8) if zone is None else np.array(zone, np.uint8)
    counts = np.zeros(max(classes * n, 1), np.int32) if counts is None else np.array(counts, np.int32)
    return lib.bs_upload_node_spread(h, n, n_zones, None if null_zone else ptr(zone), classes,
                                     None if null_counts else ptr(counts))


def _spread_pod(lib, h, P, n=None, null=False):
    n = P if n is None else n
    return lib.bs_upload_pod_spread(h, n, None if null else ptr(np.zeros(max(n, 1), np.uint32)))


def _side_cases():
    big_pref = (1 << 30) // (512 * 4) + 1   # classes x Npad (512 for one node) x 4 bytes just above the cap
    cases = _nz("node") + _nz("pod")
    f = "bs_upload_node_preferences"
    cases += [
        (f"{f}-state", break_nodes, lambda lib, h, N, P: _pref_node(lib, h, N), STATE, f"{f}: upload nodes first", TABLES),
        (f"{f}-size", None, lambda lib, h, N, P: _pref_node(lib, h, N, n=N + 1), INVAL,
         f"{f}: n_nodes differs from the node table's", PREF),
        (f"{f}-table", None, lambda lib, h, N, P: _pref_node(lib, h, N, classes=big_pref, null_w=True), INVAL,
         f"{f}: n_classes x padded nodes x 4 bytes exceeds BS_PREF_TABLE_MAX_BYTES", PREF),
        (f"{f}-null-taints", None, lambda lib, h, N, P: _pref_node(lib, h, N, taints=False), INVAL,
         f"{f}: null prefer_taints", PREF),
        (f"{f}-null-weights", None, lambda lib, h, N, P: _pref_node(lib, h, N, null_w=True), INVAL,
         f"{f}: null pref_weights", PREF),
        (f"{f}-negative", None, lambda lib, h, N, P: _pref_node(lib, h, N, weights=np.full(N, -1, np.int32)), RANGE,
         f"{f}: a preferred-affinity weight is negative", PREF),
    ]
    f = "bs_upload_pod_preferences"
    cases += [
        (f"{f}-state", break_pods, lambda lib, h, N, P: _pref_pod(lib, h, P), STATE, f"{f}: upload pods first", TABLES),
        (f"{f}-size", None, lambda lib, h, N, P: _pref_pod(lib, h, P, n=P + 1), INVAL,
         f"{f}: n_pods differs from the pod table's", PREF),
        (f"{f}-null", None, lambda lib, h, N, P: _pref_pod(lib, h, P, null=True), INVAL, f"{f}: null column", PREF),
    ]
    f = "bs_upload_node_locality"
    cases += [
        (f"{f}-state", break_nodes, lambda lib, h, N, P: _loc_node(lib, h, N), STATE, f"{f}: upload nodes first", TABLES),
        (f"{f}-size", None, lambda lib, h, N, P: _loc_node(lib, h, N, n=N + 1), INVAL,
         f"{f}: n_nodes differs from the node table's", LOC),
        (f"{f}-table", None, lambda lib, h, N, P: _loc_node(lib, h, N, n_images=(1 << 28) + 1), INVAL,
         f"{f}: n_images x ceil(n_nodes / 32) x 4 bytes exceeds BS_LOC_TABLE_MAX_BYTES", LOC),
        (f"{f}-size-range", None, lambda lib, h, N, P: _loc_node(lib, h, N, size=(-1,)), RANGE,
         f"{f}: an image size is outside [0, 2^48]", LOC),
    ]
    f = "bs_upload_pod_locality"
    cases += [
        (f"{f}-state", break_pods, lambda lib, h, N, P: _loc_pod(lib, h, P), STATE, f"{f}: upload pods first", TABLES),
        (f"{f}-size", None, lambda lib, h, N, P: _loc_pod(lib, h, P, n=P + 1), INVAL,
         f"{f}: n_pods differs from the pod table's", LOC),
        (f"{f}-table", None, lambda lib, h, N, P: _loc_pod(lib, h, P, n_classes=(1 << 30) // 512 + 1), INVAL,
         f"{f}: n_classes x padded nodes bytes exceeds BS_LOC_TABLE_MAX_BYTES", LOC),
        (f"{f}-offset0", None, lambda lib, h, N, P: _loc_pod(lib, h, P, off=(1, 1)), INVAL,
         f"{f}: class_offset[0] is not 0", LOC),
        (f"{f}-ascending", None, lambda lib, h, N, P: _loc_pod(lib, h, P, n_classes=2, off=(0, 1, 0)), INVAL,
         f"{f}: class_offset is not ascending, or a class lists more than BS_LOC_CLASS_MAX ids", LOC),
        (f"{f}-wide", None, lambda lib, h, N, P: _loc_pod(lib, h, P, off=(0, 65), ids=[0] * 65), INVAL,
         f"{f}: class_offset is not ascending, or a class lists more than BS_LOC_CLASS_MAX ids", LOC),
        (f"{f}-avoid-bit", None, lambda lib, h, N, P: _loc_pod(lib, h, P, abit=[64] * P), RANGE,
         f"{f}: an avoid bit is outside 0..63", LOC),
    ]
    f = "bs_upload_node_spread"
    cases += [
        (f"{f}-state", break_nodes, lambda lib, h, N, P: _spread_node(lib, h, N), STATE, f"{f}: upload nodes first",
         TABLES),
        (f"{f}-size", None, lambda lib, h, N, P: _spread_node(lib, h, N, n=N + 1), INVAL,
         f"{f}: n_nodes differs from the node table's", SPREAD),
        (f"{f}-zones", None, lambda lib, h, N, P: _spread_node(lib, h, N, n_zones=65), INVAL,
         f"{f}: n_zones exceeds BS_SPREAD_ZONE_MAX", SPREAD),
        (f"{f}-table", None, lambda lib, h, N, P: _spread_node(lib, h, N, classes=big_pref, null_counts=True), INVAL,
         f"{f}: n_classes x padded nodes x 4 bytes exceeds BS_SPREAD_TABLE_MAX_BYTES", SPREAD),
        (f"{f}-null-zone", None, lambda lib, h, N, P: _spread_node(lib, h, N, null_zone=True), INVAL,
         f"{f}: null zone", SPREAD),
        (f"{f}-null-counts", None, lambda lib, h, N, P: _spread_node(lib, h, N, null_counts=True), INVAL,
         f"{f}: null counts", SPREAD),
        (f"{f}-zone-id", None, lambda lib, h, N, P: _spread_node(lib, h, N, zone=[1] * N), INDEX,
         f"{f}: a zone id is >= n_zones", SPREAD),
        (f"{f}-count", None, lambda lib, h, N, P: _spread_node(lib, h, N, counts=[-1] * N), RANGE,
         f"{f}: a count is outside [0, 2^24]", SPREAD),
    ]
    f = "bs_upload_pod_spread"
    cases += [
        (f"{f}-state", break_pods, lambda lib, h, N, P: _spread_pod(lib, h, P), STATE, f"{f}: upload pods first",
         TABLES),
        (f"{f}-size", None, lambda lib, h, N, P: _spread_pod(lib, h, P, n=P + 1), INVAL,
         f"{f}: n_pods differs from the pod table's", SPREAD),
        (f"{f}-null", None, lambda lib, h, N, P: _spread_pod(lib, h, P, null=True), INVAL, f"{f}: null spread_class",
         SPREAD),
    ]
    cases += _interpod_node_cases("bs_upload_node_interpod", IPA, filter_side=False)
    cases += _interpod_node_cases("bs_upload_node_interpod_filter", IPF, filter_side=True)
    cases += _interpod_pod_cases()
    cases += _filter_pod_cases()
    return cases


def _class_cases(f, gone, call):
    """The refusals of a bs_interpod_classes table; call(lib, h, N, P, cl) uploads a side with class table cl."""
    c = lambda cl: (lambda lib, h, N, P: call(lib, h, N, P, cl))   # noqa: E731
    return [
        (f"{f}-classes-null-offset", None, c(dict(n_classes=1, null=("class_offset",))), INVAL, f"{f}: null class_offset",
         gone),
        (f"{f}-classes-offset0", None, c(dict(cl=((1, 1), (0,), (0,), (0,)))), INVAL,
         f"{f}: class_offset[0] is not 0", gone),
        (f"{f}-classes-ascending", None, c(dict(cl=((0, 1, 0), (0,), (0,), (0,)))), INVAL,
         f"{f}: class_offset is not ascending, or a class lists more than BS_IPA_CLASS_MAX entries", gone),
        (f"{f}-classes-wide", None, c(dict(cl=((0, 65), [0] * 65, [0] * 65, [0] * 65))), INVAL,
         f"{f}: class_offset is not ascending, or a class lists more than BS_IPA_CLASS_MAX entries", gone),
        (f"{f}-classes-null-term", None, c(dict(cl=((0, 1), (0,), (0,), (0,)), null=("term",))), INVAL,
         f"{f}: null term, own or match", gone),
        (f"{f}-classes-match", None, c(dict(cl=((0, 1), (0,), (0,), (2,)))), RANGE, f"{f}: a match is not 0 or 1", gone),
        (f"{f}-classes-own", None, c(dict(cl=((0, 1), (0,), ((1 << 16) + 1,), (0,)))), RANGE,
         f"{f}: an own is outside [-2^16, 2^16]", gone),
        (f"{f}-classes-twice", None, c(dict(cl=((0, 2), (0, 0), (0, 0), (0, 0)))), INVAL,
         f"{f}: a class lists one term twice", gone),
    ]


def _interpod_node_cases(f, gone, filter_side):
    def up(lib, h, t):
        return getattr(lib, f)(h, t)

    def call(**kw):
        def run(lib, h, N, P):
            t, _ = ipa_node(N, **kw)
            return up(lib, h, C.byref(t))
        return run

    def cls_call(lib, h, N, P, cl):
        t, _ = ipa_node(N, **cl)
        return up(lib, h, C.byref(t))

    limit = "BS_IPF_BOUND_MAX" if filter_side else "BS_IPA_BOUND_MAX"
    # slot totals just past each side's cap: the priority's M / S tables (16 bytes a slot), the filter's two bit planes
    slots = (dict(nv=(0xffffffff,), tkey=(0, 0)) if filter_side else dict(nv=((1 << 26) + 1,)))
    slot_msg = ("the presence planes exceed BS_IPF_TERM_MAX_BYTES" if filter_side
                else "the term tables exceed BS_IPA_TERM_MAX_BYTES")
    cases = [
        (f"{f}-null-table", None, lambda lib, h, N, P: up(lib, h, None), INVAL, f"{f}: null table", gone),
        (f"{f}-state", break_nodes, call(), STATE, f"{f}: upload nodes first", TABLES),
        (f"{f}-size", None, call(n_nodes=2), INVAL, f"{f}: n_nodes differs from the node table's", gone),
        (f"{f}-keys", None, call(n_keys=65), INVAL, f"{f}: n_keys exceeds BS_IPA_KEY_MAX", gone),
        (f"{f}-bound", None, call(n_bound=(1 << 24) + 1), INVAL, f"{f}: n_bound exceeds {limit}", gone),
        (f"{f}-null-topo", None, call(null=("topo",)), INVAL, f"{f}: null column", gone),
        (f"{f}-topo", None, call(topo=[[1]]), INDEX, f"{f}: a topo value is >= n_values", gone),
        (f"{f}-term-key", None, call(tkey=(1,)), INDEX, f"{f}: a term_key is >= n_keys", gone),
        (f"{f}-slots", None, call(**slots), INVAL, f"{f}: {slot_msg}", gone),
        (f"{f}-bound-node", None, call(bnode=(1,), bcls=(capi.IPA_NONE,)), INDEX, f"{f}: a bound_node is >= n_nodes",
         gone),
        (f"{f}-bound-class", None, call(bnode=(0,), bcls=(0,)), INDEX, f"{f}: a bound_class is >= n_classes", gone),
        (f"{f}-classes-term", None, call(cl=((0, 1), (1,), (0,), (0,))), INDEX, f"{f}: a term id is >= n_terms", gone),
    ]
    cases += _class_cases(f, gone, cls_call)
    if filter_side:
        cases.append((f"{f}-own", None, call(cl=((0, 1), (0,), (2,), (0,))), RANGE, f"{f}: an own is not 0 or 1",
                      gone))
    return cases


def _interpod_pod_cases():
    f = "bs_upload_pod_interpod"

    def call(**kw):
        def run(lib, h, N, P):
            t, _ = ipa_pods(P, **kw)
            return lib.bs_upload_pod_interpod(h, C.byref(t))
        return run

    def cls_call(lib, h, N, P, cl):
        t, _ = ipa_pods(P, **cl)
        return lib.bs_upload_pod_interpod(h, C.byref(t))

    cases = [
        (f"{f}-null-table", None, lambda lib, h, N, P: lib.bs_upload_pod_interpod(h, None), INVAL, f"{f}: null table",
         IPA),
        (f"{f}-state", break_pods, call(), STATE, f"{f}: upload pods first", TABLES),
        (f"{f}-size", None, call(n_pods=11), INVAL, f"{f}: n_pods differs from the pod table's", IPA),
        (f"{f}-null-class", None, call(null=("pod_class",)), INVAL, f"{f}: null pod_class", IPA),
        (f"{f}-table", None, call(n_classes=(1 << 18) + 1), INVAL,
         f"{f}: n_classes x padded nodes x 8 bytes exceeds BS_IPA_TABLE_MAX_BYTES", IPA),
        (f"{f}-pod-class", None, call(pcls=[1] * 10), INDEX, f"{f}: a pod_class is >= n_classes", IPA),
    ]
    return cases + _class_cases(f, IPA, cls_call)


def _filter_pod_cases():
    f = "bs_upload_pod_interpod_filter"

    def call(**kw):
        def run(lib, h, N, P):
            t, _ = ipf_pods(P, **kw)
            return lib.bs_upload_pod_interpod_filter(h, C.byref(t))
        return run

    asc = "class_offset is not ascending, or a class lists more than BS_IPF_CLASS_MAX entries"
    return [
        (f"{f}-null-table", None, lambda lib, h, N, P: lib.bs_upload_pod_interpod_filter(h, None), INVAL,
         f"{f}: null table", IPF),
        (f"{f}-state", break_pods, call(), STATE, f"{f}: upload pods first", TABLES),
        (f"{f}-size", None, call(n_pods=11), INVAL, f"{f}: n_pods differs from the pod table's", IPF),
        (f"{f}-null-class", None, call(null=("pod_class",)), INVAL, f"{f}: null pod_class", IPF),
        (f"{f}-null-offset", None, call(null=("class_offset",)), INVAL, f"{f}: null class_offset or self_match", IPF),
        (f"{f}-table", None, call(n_classes=(1 << 30) // (3 * 64) + 1),
         INVAL, f"{f}: 3 x n_classes x padded nodes / 8 bytes exceeds BS_IPF_TABLE_MAX_BYTES", IPF),
        (f"{f}-offset0", None, call(off=(1, 1)), INVAL, f"{f}: class_offset[0] is not 0", IPF),
        (f"{f}-ascending", None, call(off=(0, 1, 0), self_match=(0, 0)), INVAL, f"{f}: {asc}", IPF),
        (f"{f}-wide", None, call(off=(0, 65), term=[0] * 65, role=[0] * 65), INVAL, f"{f}: {asc}", IPF),
        (f"{f}-null-term", None, call(null=("term",)), INVAL, f"{f}: null term or role", IPF),
        (f"{f}-role", None, call(role=(3,)), INVAL,
         f"{f}: a role is not BS_IPF_AFFINITY, BS_IPF_ANTI or BS_IPF_EXISTING", IPF),
        (f"{f}-self-match", None, call(self_match=(2,)), RANGE, f"{f}: a self_match is not 0 or 1", IPF),
        (f"{f}-pod-class", None, call(pcls=[1] * 10), INDEX, f"{f}: a pod_class is >= n_classes", IPF),
    ]


SIDE_CASES = _side_cases()


@pytest.mark.parametrize("case", SIDE_CASES, ids=[c[0] for c in SIDE_CASES])
def test_side_upload_refusal(eng, case):
    _, prepare, call, code, text, gone = case
    if prepare:
        prepare(eng)
    rc = call(eng.lib, eng.h, eng.snap.nodes.n, eng.snap.pods.n)
    assert (rc, last_error(eng)) == (code, text)
    assert evaluate(eng) == (STATE, gone)


# ---- bs_evaluate's and bs_replay_priority's checks --------------------------------------------------------------
def _bigger_nodes(eng):
    """513 nodes: Npad doubles to 1024 under a pod side checked against 512."""
    eng.upload_nodes(S.NodeTable.empty(513, L))
    node_sides(eng, 513)


def _check_cases(who):
    w = who

    def run(*steps):   # a step may be an upload that fails on purpose: the round's answer is what is checked
        def go(e):
            for s in steps:
                s(e)
        return go

    P = 10   # every array is built inside its step, so its pointer is taken while the test runs

    def ipa_pod(**kw):
        def go(e):
            t, _ = ipa_pods(P, **kw)
            return e.lib.bs_upload_pod_interpod(e.h, C.byref(t))
        return go

    def ipf_pod(**kw):
        def go(e):
            t, _ = ipf_pods(P, **kw)
            return e.lib.bs_upload_pod_interpod_filter(e.h, C.byref(t))
        return go

    def loc_pod(**kw):
        return lambda e: _loc_pod(e.lib, e.h, P, **kw)

    cases = [
        ("loc-state", run(lambda e: e.lib.bs_upload_pod_locality(e.h, P, None, 0, None, None, ptr(np.zeros(P, np.uint8)))),
         STATE, f"{w}: a non-zero ImageLocality weight needs the node and pod image columns"),
        ("loc-class", run(loc_pod(cls=[1] * P)), INDEX, f"{w}: a pod's image class is outside the uploaded classes"),
        ("loc-image", run(loc_pod(ids=(1,))), INDEX,
         f"{w}: an image class lists an id outside the node side's image dictionary"),
        ("loc-table", run(lambda e: loc_pod(n_classes=1 << 21, off=np.zeros((1 << 21) + 1, np.uint32), ids=())(e),
                          _bigger_nodes),
         INVAL, f"{w}: n_classes x padded nodes bytes exceeds BS_LOC_TABLE_MAX_BYTES"),
        ("loc-avoid", run(lambda e: e.set_locality_weights(0, 1), loc_pod(avoid=False)), STATE,
         f"{w}: a non-zero NodePreferAvoidPods weight needs the node and pod avoid columns"),
    ]
    if who == "bs_replay_priority":
        return cases + [
            ("nz-state", run(lambda e: e.lib.bs_upload_pod_nonzero(e.h, P, None)), STATE,
             f"{w}: upload both non-zero request columns first"),
        ]
    return cases + [
        ("nz-state", run(lambda e: e.lib.bs_upload_pod_nonzero(e.h, P, None)), STATE, NZ),
        ("pref-state", run(lambda e: e.lib.bs_upload_pod_preferences(e.h, P, None, None)), STATE, PREF),
        ("pref-class", run(lambda e: e.lib.bs_upload_pod_preferences(e.h, P, ptr(np.zeros(P, np.uint64)),
                                                                     ptr(np.ones(P, np.uint32)))), INDEX,
         f"{w}: a pod's preference class is outside the uploaded weight table"),
        ("spread-state", run(lambda e: e.lib.bs_upload_pod_spread(e.h, P, None)), STATE, SPREAD),
        ("spread-class", run(lambda e: e.lib.bs_upload_pod_spread(e.h, P, ptr(np.ones(P, np.uint32)))), INDEX,
         f"{w}: a pod's spread class is outside the uploaded count table"),
        ("ipa-state", run(lambda e: e.lib.bs_upload_pod_interpod(e.h, None)), STATE, IPA),
        ("ipa-term", run(ipa_pod(cl=((0, 1), (1,), (1,), (1,)))), INDEX,
         f"{w}: a pod class's term is outside the node side's term dictionary"),
        ("ipa-table", run(lambda e: ipa_pod(cl=(np.zeros((1 << 18) + 1, np.uint32), (), (), ()))(e), _bigger_nodes),
         INVAL,
         f"{w}: pod n_classes x padded nodes x 8 bytes exceeds BS_IPA_TABLE_MAX_BYTES"),
        ("ipf-state", run(lambda e: e.lib.bs_upload_pod_interpod_filter(e.h, None)), STATE, IPF),
        ("ipf-term", run(ipf_pod(term=(1,))), INDEX,
         f"{w}: a filter class's term is outside the node side's term dictionary"),
        ("ipf-table", run(lambda e: ipf_pod(off=np.zeros(4000001, np.uint32), term=(), role=(),
                                                self_match=np.zeros(4000000, np.uint8))(e), _bigger_nodes), INVAL,
         f"{w}: 3 x filter n_classes x padded nodes / 8 bytes exceeds BS_IPF_TABLE_MAX_BYTES"),
    ]


EVAL_CASES = _check_cases("bs_evaluate")
REPLAY_CASES = _check_cases("bs_replay_priority")


@pytest.mark.parametrize("case", EVAL_CASES, ids=[c[0] for c in EVAL_CASES])
def test_evaluate_check(eng, case):
    _, prepare, code, text = case
    prepare(eng)
    assert evaluate(eng) == (code, text)


@pytest.mark.parametrize("case", REPLAY_CASES, ids=[c[0] for c in REPLAY_CASES])
def test_replay_priority_check(eng, case):
    _, prepare, code, text = case
    eng.set_interpod_filter(False)
    eng.set_node_priority_weights(0, 0)
    eng.set_spread_weight(0)
    eng.set_interpod_weight(0)
    assert replay_priority(eng) == (OK, "")
    prepare(eng)
    assert replay_priority(eng) == (code, text)
