"""A second, independent restatement of the InterPodAffinity priority (include/bsched.h bs_set_interpod_weight) in pure
Python over small objects, written from kube-scheduler v1.17's interpod_affinity.go [upstream, from memory]
(processTerm, processTerms, processExistingPod, CalculateInterPodAffinityPriorityReduce) without looking at the C
restatement: each matching term adds its weight to every node that shares the topology value of the fixed pod's node,
compared label by label.  Python floats are binary64 and CPython never fuses a multiply and an add, so the arithmetic
is Go's.  The resource part of the score is tests/pyref_ratio_priority.py's.

pack() is the other half: the packing rules of the plugin's PackInterPodAffinity restated over the same objects, which
turn them into the engine's columns (bs_upload_node_interpod / bs_upload_pod_interpod)."""
from dataclasses import dataclass, field

from pyref import Node, i64, resource_from
from pyref_priority import INT64_MIN, fits
from pyref_ratio_priority import total

IPA_NONE = 0xFFFFFFFF
TOPO_NONE = 0xFFFFFFFF
CLASS_MAX = 64


class InvalidSelector(Exception):
    """metav1.LabelSelectorAsSelector failed."""


@dataclass
class Selector:
    """metav1.LabelSelector: match_labels {key: value} and match_expressions [(key, op, [values])]."""
    match_labels: dict = field(default_factory=dict)
    match_expressions: list = field(default_factory=list)


@dataclass
class Term:
    """v1.PodAffinityTerm: selector None is a nil selector; namespaces () means the defining pod's namespace."""
    selector: Selector = None
    namespaces: tuple = ()
    key: str = ""


@dataclass
class PodObj:
    namespace: str = "default"
    labels: dict = field(default_factory=dict)
    required: list = field(default_factory=list)     # [Term]: required pod affinity
    preferred: list = field(default_factory=list)    # [(weight, Term)]: preferred pod affinity
    anti: list = field(default_factory=list)         # [(weight, Term)]: preferred pod anti-affinity
    terminating: bool = False
    node: int = None                                 # a bound pod's node


def requirements(sel):
    """LabelSelectorAsSelector: the requirements (matchLabels as "=") sorted by key, operator and values;
    InvalidSelector when one fails to convert."""
    reqs = [(k, "=", (v,)) for k, v in sel.match_labels.items()]
    for k, op, vals in sel.match_expressions:
        if op in ("In", "NotIn"):
            if not vals:
                raise InvalidSelector(f"{op} without values")
        elif op in ("Exists", "DoesNotExist"):
            if vals:
                raise InvalidSelector(f"{op} with values")
        else:
            raise InvalidSelector(f"operator {op}")
        reqs.append((k, op, tuple(sorted(vals))))
    return sorted(reqs)


def selector_matches(sel, labels):
    """A nil selector matches nothing, an empty one everything."""
    if sel is None:
        return False
    for k, op, vals in requirements(sel):
        has = k in labels
        if op in ("=", "In") and not (has and labels[k] in vals):
            return False
        if op == "NotIn" and has and labels[k] in vals:
            return False
        if op == "Exists" and not has:
            return False
        if op == "DoesNotExist" and has:
            return False
    return True


def term_namespaces(term, defining):
    return set(term.namespaces) if term.namespaces else {defining.namespace}


def pod_matches_term(pod, term, defining):
    """processTerm's match: the selector converts first (failing whatever the namespaces), then
    PodMatchesTermsNamespaceAndSelector."""
    sel = selector_matches(term.selector, pod.labels)
    return pod.namespace in term_namespaces(term, defining) and sel


def same_topology(labels, a, b, key):
    """NodesHaveSameTopologyKey: both nodes carry the key, with one value; an empty key never holds."""
    return key != "" and key in labels[a] and key in labels[b] and labels[a][key] == labels[b][key]


def process_term(counts, labels, term, defining, to_check, fixed_node, weight):
    if pod_matches_term(to_check, term, defining):
        for n in range(len(labels)):
            if same_topology(labels, n, fixed_node, term.key):
                counts[n] += weight


def raw_scores(pod, bound, labels, hard=1):
    """{node: raw} of a pending pod over every node: processExistingPod for each bound pod; InvalidSelector when
    upstream would fail the pod's score."""
    counts = [0] * len(labels)
    for e in bound:
        # the pod's own terms against the bound pod
        for w, t in pod.preferred:
            process_term(counts, labels, t, pod, e, e.node, w)
        for w, t in pod.anti:
            process_term(counts, labels, t, pod, e, e.node, -w)
        # the bound pod's terms against the pod
        if hard > 0:
            for t in e.required:
                process_term(counts, labels, t, e, pod, e.node, hard)
        for w, t in e.preferred:
            process_term(counts, labels, t, e, pod, e.node, w)
        for w, t in e.anti:
            process_term(counts, labels, t, e, pod, e.node, -w)
    return dict(enumerate(counts))


def reduce(raw):
    """CalculateInterPodAffinityPriorityReduce over the filtered nodes: {node: raw} -> {node: score}."""
    mx = mn = 0
    for v in raw.values():
        mx = max(mx, v)
        mn = min(mn, v)
    out = {}
    for n, v in raw.items():
        f = 0.0
        if mx - mn > 0:
            f = 100.0 * (float(v - mn) / float(mx - mn))
        out[n] = int(f)
    return out


def priority_rows(snap, node_nz, pod_nz, K, pending, bound, labels, w_ipa, hard=1,
                  setting=(0, ((0, 100), (100, 0)), [0] * 4), weights=(1, 0, 1), pods=None):
    """Per pod: [(node, score), ...] of its fitting nodes, score descending then node ascending, padded to K with
    (-1, INT64_MIN).  pending[p] / bound / labels: the objects behind the snapshot's pods and nodes."""
    nt, pt = snap.nodes, snap.pods
    if len(setting[2]) != nt.lanes:
        setting = (setting[0], setting[1], list(setting[2]) + [0] * (nt.lanes - len(setting[2]))) + tuple(setting[3:])
    nodes = [Node(nt, i) for i in range(nt.n)]
    aff_bits = getattr(snap, "aff_bits", None)
    out = []
    for p in (range(pt.n) if pods is None else pods):
        fit = [i for i in range(nt.n) if fits(nodes[i], pt, p, i, aff_bits, nt.lanes)]
        try:
            raw = raw_scores(pending[p], bound, labels, hard)
        except InvalidSelector:
            raw = {i: 0 for i in range(nt.n)}   # the score fails: the pod scores 0 everywhere
        ipa = reduce({i: raw[i] for i in fit})
        req = resource_from(pt.req[:, p], int(pt.req_present[p]), nt.lanes)
        pnz = (int(pod_nz[0][p]), int(pod_nz[1][p]))
        cand = []
        for i in fit:
            s = total(setting, weights, nodes[i], (int(node_nz[0][i]), int(node_nz[1][i])), pnz, req)
            cand.append((i64(s + w_ipa * ipa[i]), i))
        cand.sort(key=lambda t: (-t[0], t[1]))
        row = [(i, s) for s, i in cand[:K]]
        out.append(row + [(-1, INT64_MIN)] * (K - len(row)))
    return out


# ---- the packing rules ----

def _own_terms(pod, hard, bound_side):
    """[(term, signed weight)] of the terms the pod's processing reads, in order: required affinity (a bound pod's,
    while hard > 0), preferred affinity, preferred anti-affinity."""
    out = [(t, hard) for t in pod.required] if bound_side and hard > 0 else []
    return out + [(t, w) for w, t in pod.preferred] + [(t, -w) for w, t in pod.anti]


def pack(pending, bound, labels, hard=1):
    """The columns and dictionaries PackInterPodAffinity builds: a dict with node = (n_values, topo, term_key,
    bound_node, bound_class, classes), pods = (pod_class, classes), and the dictionaries keys, values (per key),
    terms ((sorted namespaces, requirements, key)), bound_classes and pod_classes (each a tuple of (term, own, match)).

    Keys and terms are numbered in order of first appearance over the bound pods' terms, then the pending pods'; a
    term's identity is its resolved, sorted namespaces, its selector's requirements and its key.  A term with an empty
    key never matches a node and is left out, as is a term whose selector fails to convert.  A key's values are
    numbered in order of first appearance over the nodes.  A pod lists (t, own, match) for each term it owns (own = its
    summed signed weights) or that it matches among the other side's terms; a pod without entries has no class.
    Classes are numbered in order of first appearance.  A pending pod gets no class (it scores 0) when a bound pod's
    processed term fails to convert, or when one of its own terms does and some pod is bound."""
    keys, terms = {}, {}
    invalid_bound = False

    def own_of(pod, bound_side):
        own, bad = {}, False
        for t, w in _own_terms(pod, hard, bound_side):
            try:
                reqs = tuple(requirements(t.selector)) if t.selector is not None else None
            except InvalidSelector:
                bad = True
                continue
            if t.key == "":
                continue
            keys.setdefault(t.key, len(keys))
            tid = terms.setdefault((tuple(sorted(term_namespaces(t, pod))), reqs, t.key), (len(terms), t, pod))[0]
            own[tid] = own.get(tid, 0) + w
        return own, bad

    bown = []
    for e in bound:
        o, bad = own_of(e, True)
        invalid_bound |= bad
        bown.append(o)
    pown, pbad = [], []
    for p in pending:
        o, bad = own_of(p, False)
        pown.append(o)
        pbad.append(bad and len(bound) > 0)
    by_id = {v[0]: v for v in terms.values()}
    b_terms = sorted({t for o in bown for t in o})
    p_terms = sorted({t for o in pown for t in o})

    def entries(pod, own, other_terms):
        m = {t for t in other_terms if pod_matches_term(pod, by_id[t][1], by_id[t][2])}
        ent = tuple((t, own.get(t, 0), 1 if t in m else 0) for t in sorted(set(own) | m))
        ent = tuple(x for x in ent if x[1] != 0 or x[2] != 0)
        if len(ent) > CLASS_MAX:
            raise ValueError("a pod lists more than BS_IPA_CLASS_MAX terms")
        return ent

    def classify(rows):
        classes, ids = {}, []
        for ent in rows:
            ids.append(IPA_NONE if ent is None or not ent else classes.setdefault(ent, len(classes)))
        return ids, list(classes)

    bound_class, bclasses = classify([entries(e, o, p_terms) for e, o in zip(bound, bown)])
    pod_rows = [None if (invalid_bound or bad) else entries(p, o, b_terms) for p, o, bad in zip(pending, pown, pbad)]
    pod_class, pclasses = classify(pod_rows)
    key_list = sorted(keys, key=keys.get)
    values = []
    topo = []
    for k in key_list:
        vals = {}
        row = []
        for lab in labels:
            row.append(vals.setdefault(lab[k], len(vals)) if k in lab else TOPO_NONE)
        values.append(list(vals))
        topo.append(row)
    term_list = sorted(terms.items(), key=lambda kv: kv[1][0])
    term_key = [keys[k[2]] for k, _ in term_list]

    def table(classes):
        off, tt, oo, mm = [0], [], [], []
        for ent in classes:
            for t, o, m in ent:
                tt.append(t)
                oo.append(o)
                mm.append(m)
            off.append(len(tt))
        return off, tt, oo, mm

    return dict(node=([len(v) for v in values], topo, term_key, [e.node for e in bound], bound_class,
                      table(bclasses)),
                pods=(pod_class, table(pclasses)), keys=key_list, values=values, terms=[k for k, _ in term_list],
                bound_classes=bclasses, pod_classes=pclasses)
