"""A second, independent restatement of the SelectorSpread priority (include/bsched.h bs_set_spread_weight) in pure
Python over the Go-like objects of tests/pyref.py, written from kube-scheduler v1.17's selector_spreading.go
[upstream, from memory] without looking at the C restatement.  Python floats are binary64 and CPython never fuses a
multiply and an add, so the arithmetic is Go's.  The resource part of the score is tests/pyref_ratio_priority.py's, and
the TaintToleration and NodeAffinity terms tests/pyref_node_priority.py's.  Python ints are masked to int64 where Go
would wrap."""
from pyref import Node, i64, resource_from
from pyref_node_priority import affinity_count, normalize_reduce, taint_count
from pyref_priority import INT64_MIN, fits
from pyref_ratio_priority import total

SPREAD_NONE = 0xFFFFFFFF
ZONE_NONE = 0xFF
ZONE_WEIGHTING = 2.0 / 3.0


def spread_reduce(counts, zone_of):
    """CalculateSpreadPriorityReduce over the filtered nodes: counts = {node: count}, zone_of = {node: zone id or
    None}; returns {node: score}."""
    max_by_node = 0
    by_zone = {}
    for i, c in counts.items():
        max_by_node = max(max_by_node, c)
        z = zone_of[i]
        if z is not None:
            by_zone[z] = by_zone.get(z, 0) + c
    max_by_zone = max(by_zone.values(), default=0)
    have_zones = len(by_zone) != 0
    out = {}
    for i, c in counts.items():
        z = zone_of[i]
        zoned = have_zones and z is not None
        out[i] = node_score(max_by_node, c, zoned, max_by_zone, by_zone[z] if zoned else 0)
    return out


def node_score(max_by_node, count, zoned, max_by_zone, zone_count):
    """The reduce's score of one node: fScore, blended with the zone score when the node is zoned."""
    f = 100.0
    if max_by_node > 0:
        f = 100.0 * (float(max_by_node - count) / float(max_by_node))
    if zoned:
        zs = 100.0
        if max_by_zone > 0:
            zs = 100.0 * (float(max_by_zone - zone_count) / float(max_by_zone))
        f = f * (1.0 - ZONE_WEIGHTING) + ZONE_WEIGHTING * zs
    return int(f)


def priority_rows(snap, node_nz, pod_nz, K, spread, w_spread, setting=(0, ((0, 100), (100, 0)), [0] * 4),
                  weights=(1, 0, 1), prefs=None, pref_weights=(0, 0), pods=None):
    """Per pod: [(node, score), ...] of its fitting nodes, score descending then node ascending, padded to K with
    (-1, INT64_MIN).  spread = ((zone [N], counts [C, N]), spread_class [P]); prefs as pyref_node_priority's."""
    nt, pt = snap.nodes, snap.pods
    (zone, table), cls = spread
    if len(setting[2]) != nt.lanes:
        setting = (setting[0], setting[1], list(setting[2]) + [0] * (nt.lanes - len(setting[2]))) + tuple(setting[3:])
    nodes = [Node(nt, i) for i in range(nt.n)]
    aff_bits = getattr(snap, "aff_bits", None)
    zone_of = {i: (None if int(zone[i]) == ZONE_NONE else int(zone[i])) for i in range(nt.n)}
    out = []
    for p in (range(pt.n) if pods is None else pods):
        fit = [i for i in range(nt.n) if fits(nodes[i], pt, p, i, aff_bits, nt.lanes)]
        c = int(cls[p])
        ss = spread_reduce({i: (0 if c == SPREAD_NONE else int(table[c][i])) for i in fit}, zone_of)
        tt = na = None
        if prefs is not None:
            taints, ptab, tol, pcls = prefs
            tt = normalize_reduce({i: taint_count(taints[i], tol[p]) for i in fit}, True)
            na = normalize_reduce({i: affinity_count(ptab, pcls[p], i) for i in fit}, False)
        req = resource_from(pt.req[:, p], int(pt.req_present[p]), nt.lanes)
        pnz = (int(pod_nz[0][p]), int(pod_nz[1][p]))
        cand = []
        for i in fit:
            s = total(setting, weights, nodes[i], (int(node_nz[0][i]), int(node_nz[1][i])), pnz, req)
            if prefs is not None:
                s += pref_weights[0] * tt[i] + pref_weights[1] * na[i]
            cand.append((i64(s + w_spread * ss[i]), i))
        cand.sort(key=lambda t: (-t[0], t[1]))
        row = [(i, s) for s, i in cand[:K]]
        out.append(row + [(-1, INT64_MIN)] * (K - len(row)))
    return out
