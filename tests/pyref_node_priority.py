"""A second, independent restatement of the TaintToleration and preferred NodeAffinity priorities (include/bsched.h
bs_set_node_priority_weights) in pure Python over the Go-like objects of tests/pyref.py, written from kube-scheduler
v1.17's taint_toleration.go, node_affinity.go and NormalizeReduce [upstream, from memory] without looking at the C
restatement.  The resource part of the score is tests/pyref_ratio_priority.py's.  Python ints are masked to int64
where Go would wrap."""
from pyref import Node, i64, resource_from
from pyref_priority import INT64_MIN, fits
from pyref_ratio_priority import total

PREF_NONE = 0xFFFFFFFF


def taint_count(prefer_taints_n, prefer_tol_p):
    """CalculateTaintTolerationPriorityMap: intolerable PreferNoSchedule taints of the node."""
    return bin(int(prefer_taints_n) & ~int(prefer_tol_p) & ((1 << 64) - 1)).count("1")


def affinity_count(pref_weights, cls, i):
    """CalculateNodeAffinityPriorityMap: the summed weights of the pod's matching preferred terms (per class)."""
    return 0 if int(cls) == PREF_NONE else int(pref_weights[int(cls)][i])


def normalize_reduce(counts, reverse):
    """NormalizeReduce(MaxNodeScore = 100, reverse) over the counts of the filtered nodes."""
    mx = max(counts.values(), default=0)
    out = {}
    for i, c in counts.items():
        s = 100 if mx == 0 else (100 * c) // mx   # counts are >= 0: floor is truncation
        out[i] = (100 - s if mx else 100) if reverse else (s if mx else 0)
    return out


def priority_rows(snap, node_nz, pod_nz, K, prefs, pref_weights=(0, 0), setting=(0, ((0, 100), (100, 0)), [0] * 4),
                  weights=(1, 0, 1), pods=None):
    """Per pod: [(node, score), ...] of its fitting nodes, score descending then node ascending, padded to K with
    (-1, INT64_MIN).  prefs = (prefer_taints, pref_weights table, prefer_tol, pref_class); pref_weights = the two
    weights (TaintToleration, NodeAffinity); setting = the ratio setting (weight 0 = off)."""
    nt, pt = snap.nodes, snap.pods
    taints, table, tol, cls = prefs
    w_taint, w_naff = pref_weights
    if len(setting[2]) != nt.lanes:
        setting = (setting[0], setting[1], list(setting[2]) + [0] * (nt.lanes - len(setting[2]))) + tuple(setting[3:])
    nodes = [Node(nt, i) for i in range(nt.n)]
    aff_bits = getattr(snap, "aff_bits", None)
    out = []
    for p in (range(pt.n) if pods is None else pods):
        fit = [i for i in range(nt.n) if fits(nodes[i], pt, p, i, aff_bits, nt.lanes)]
        tt = normalize_reduce({i: taint_count(taints[i], tol[p]) for i in fit}, True)
        na = normalize_reduce({i: affinity_count(table, cls[p], i) for i in fit}, False)
        req = resource_from(pt.req[:, p], int(pt.req_present[p]), nt.lanes)
        pnz = (int(pod_nz[0][p]), int(pod_nz[1][p]))
        cand = []
        for i in fit:
            s = total(setting, weights, nodes[i], (int(node_nz[0][i]), int(node_nz[1][i])), pnz, req)
            cand.append((i64(s + w_taint * tt[i] + w_naff * na[i]), i))
        cand.sort(key=lambda t: (-t[0], t[1]))
        row = [(i, s) for s, i in cand[:K]]
        out.append(row + [(-1, INT64_MIN)] * (K - len(row)))
    return out
