"""TEST INFRASTRUCTURE — kube-scheduler v1.17's MatchInterPodAffinity filter restated from objects [upstream, from
memory], and a packer from the objects to the engine's columns (include/bsched.h bs_upload_node_interpod_filter,
bs_upload_pod_interpod_filter).

The restatement builds upstream's topology-pair maps under the names of the functions that build them
(getTPMapMatchingExistingAntiAffinity, getTPMapMatchingIncomingAffinityAntiAffinity) and checks them the way
satisfiesExistingPodsAntiAffinity and satisfiesPodsAffinityAntiAffinity do: keyed by (key, value), not by term.  The
packer resolves the same objects into the per-term dictionary, so tests/interpod_filter_ref.c over its columns and
verdict() here must agree.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

INVALID = "invalid"   # a selector that LabelSelectorAsSelector rejects: matches no pod
IPF_NONE = 0xFFFFFFFF
TOPO_NONE = 0xFFFFFFFF
AFFINITY, ANTI, EXISTING = range(3)


@dataclass
class Term:
    selector: object            # None (nil: nothing), {} (everything), {label: value} (matchLabels) or INVALID
    key: str                    # topologyKey; "" is a key no node carries
    namespaces: list = field(default_factory=list)   # empty: the namespace of the pod that defines the term


@dataclass
class Pod:
    name: str
    ns: str = "default"
    labels: dict = field(default_factory=dict)
    node: str = None            # the node of a bound pod
    affinity: list = field(default_factory=list)   # required pod affinity terms
    anti: list = field(default_factory=list)       # required pod anti-affinity terms
    terminating: bool = False   # counts like any other pod


def selector_matches(sel, labels) -> bool:
    if sel is None or sel == INVALID:
        return False
    return all(labels.get(k) == v for k, v in sel.items())


def pod_matches_term(pod: Pod, term: Term, owner_ns: str) -> bool:
    """PodMatchesTermsNamespaceAndSelector with the term's namespaces defaulted to its owner's."""
    return pod.ns in (term.namespaces or [owner_ns]) and selector_matches(term.selector, pod.labels)


def getTPMapMatchingExistingAntiAffinity(pod: Pod, existing, nodes) -> set:
    pairs = set()
    for e in existing:
        labels = nodes.get(e.node)
        if labels is None:
            continue
        for w in e.anti:
            if pod_matches_term(pod, w, e.ns) and w.key in labels:
                pairs.add((w.key, labels[w.key]))
    return pairs


def getTPMapMatchingIncomingAffinityAntiAffinity(pod: Pod, existing, nodes):
    aff, anti = set(), set()
    for e in existing:
        labels = nodes.get(e.node)
        if labels is None:
            continue
        if pod.affinity and all(pod_matches_term(e, t, pod.ns) for t in pod.affinity):   # podMatchesAllAffinityTermProperties
            for t in pod.affinity:
                if t.key in labels:
                    aff.add((t.key, labels[t.key]))
        for u in pod.anti:
            if pod_matches_term(e, u, pod.ns) and u.key in labels:
                anti.add((u.key, labels[u.key]))
    return aff, anti


def satisfiesExistingPodsAntiAffinity(node_labels: dict, pairs: set) -> bool:
    return not any((k, v) in pairs for k, v in node_labels.items())


def satisfiesPodsAffinityAntiAffinity(pod: Pod, node_labels: dict, aff: set, anti: set) -> str:
    """None when the node passes, else "A" or "N"."""
    if pod.affinity:
        ok = all(t.key in node_labels and (t.key, node_labels[t.key]) in aff for t in pod.affinity)
        if not ok and not (not aff and all(pod_matches_term(pod, t, pod.ns) for t in pod.affinity)):
            return "A"
    if pod.anti and any(u.key in node_labels and (u.key, node_labels[u.key]) in anti for u in pod.anti):
        return "N"
    return None


def verdict(pod: Pod, node: str, nodes: dict, existing) -> str:
    """None when pod passes node under InterPodAffinityMatches, else the failing step: "E", "A" or "N"."""
    labels = nodes[node]
    if not satisfiesExistingPodsAntiAffinity(labels, getTPMapMatchingExistingAntiAffinity(pod, existing, nodes)):
        return "E"
    if not pod.affinity and not pod.anti:
        return None
    aff, anti = getTPMapMatchingIncomingAffinityAntiAffinity(pod, existing, nodes)
    return satisfiesPodsAffinityAntiAffinity(pod, labels, aff, anti)


def pack(nodes: dict, existing, pending):
    """(node side, pod side) of the engine for the node list (name -> labels, in order), the existing pods and the
    pending pods (in order).  Existing pods on a node outside `nodes` are left out."""
    names = list(nodes)
    keys, values = {}, []
    term_key, boff, bterm, bown, bmatch, bnode, bcls = [], [0], [], [], [], [], []

    def key_id(k):
        if k not in keys:
            keys[k] = len(keys)
            vals = {}
            for n in names:
                if k in nodes[n]:
                    vals.setdefault(nodes[n][k], len(vals))
            values.append(vals)
        return keys[k]

    def new_term(k):
        term_key.append(key_id(k))
        return len(term_key) - 1

    bound = [e for e in existing if e.node in nodes]
    entries = [dict() for _ in bound]   # per bound pod: term -> [own, match]
    # the existing pods' required anti-affinity terms, one dictionary term per distinct resolved term
    owned = {}
    for i, e in enumerate(bound):
        for w in e.anti:
            ident = (tuple(sorted(w.namespaces or [e.ns])), repr(w.selector), w.key)
            if ident not in owned:
                owned[ident] = (new_term(w.key), Term(w.selector, w.key, list(w.namespaces or [e.ns])))
            entries[i].setdefault(owned[ident][0], [0, 0])[0] = 1
    poff, pterm, prole, pself, pod_class = [0], [], [], [], []
    for p in pending:
        ent = []
        for t, w in owned.values():
            if pod_matches_term(p, w, p.ns):   # w carries its owner's namespaces
                ent.append((t, EXISTING))
        for a in p.affinity:   # the set's terms: a bound pod matches each when it matches all of them
            t = new_term(a.key)
            ent.append((t, AFFINITY))
            for i, e in enumerate(bound):
                if all(pod_matches_term(e, x, p.ns) for x in p.affinity):
                    entries[i].setdefault(t, [0, 0])[1] = 1
        for u in p.anti:
            t = new_term(u.key)
            ent.append((t, ANTI))
            for i, e in enumerate(bound):
                if pod_matches_term(e, u, p.ns):
                    entries[i].setdefault(t, [0, 0])[1] = 1
        if not ent:
            pod_class.append(IPF_NONE)
            continue
        pod_class.append(len(poff) - 1)
        pterm += [t for t, _ in ent]
        prole += [r for _, r in ent]
        poff.append(len(pterm))
        pself.append(1 if p.affinity and all(pod_matches_term(p, x, p.ns) for x in p.affinity) else 0)
    for i, e in enumerate(bound):
        bnode.append(names.index(e.node))
        if not entries[i]:
            bcls.append(IPF_NONE)
            continue
        bcls.append(len(boff) - 1)
        for t, (o, m) in entries[i].items():
            bterm.append(t); bown.append(o); bmatch.append(m)
        boff.append(len(bterm))
    key_list = list(keys)
    topo = np.array([[values[k].get(nodes[n].get(kn), TOPO_NONE) if kn in nodes[n] else TOPO_NONE for n in names]
                     for k, kn in enumerate(key_list)], np.uint32).reshape(len(key_list), len(names))
    node = (np.array([max(len(v), 1) for v in values], np.uint32), topo, np.array(term_key, np.uint32),
            np.array(bnode, np.uint32), np.array(bcls, np.uint32),
            (np.array(boff, np.uint32), np.array(bterm, np.uint32), np.array(bown, np.int32), np.array(bmatch, np.uint8)))
    pods = (np.array(pod_class, np.uint32), (np.array(poff, np.uint32), np.array(pterm, np.uint32),
                                             np.array(prole, np.uint8), np.array(pself, np.uint8)))
    return node, pods
