"""A second, independent restatement of the RequestedToCapacityRatio priority (include/bsched.h bs_set_ratio_priority)
in pure Python over the Go-like objects of tests/pyref.py, written from kube-scheduler v1.17's
requested_to_capacity_ratio.go [upstream, from memory] without looking at the C restatement: the priority lists and a
chooser for tests/pyref_replay_priority.py's walk.  Python floats are IEEE binary64 like Go's float64; Python ints are
masked to int64 where Go would wrap.  Python's round() rounds half to even, so math.Round is written out."""
import math

from pyref import Node, i64, resource_from
from pyref_priority import INT64_MIN, fits, score as priority_score
from pyref_replay_priority import PriorityChooser


def _trunc_div(a, b):   # Go's int64 division truncates toward zero; MinInt64 / -1 wraps back to MinInt64
    q = abs(a) // abs(b)
    return i64(q if (a >= 0) == (b >= 0) else -q)


def broken_linear(shape, p):
    """buildBrokenLinearFunction: shape is [(utilization, score), ...], utilization ascending."""
    for i, (u, s) in enumerate(shape):
        if p <= u:
            if i == 0:
                return shape[0][1]
            u0, s0 = shape[i - 1]
            return s0 + _trunc_div((s - s0) * (p - u0), u - u0)
    return shape[-1][1]


def utilization(requested, capacity):
    """maxUtilization - (capacity - requested) * maxUtilization / capacity, 100 when capacity is 0 or exceeded."""
    if capacity == 0 or requested > capacity:
        return 100
    return i64(100 - _trunc_div(i64(i64(capacity - requested) * 100), capacity))


def go_round(x):
    """math.Round for x >= 0: half away from zero.  x - floor(x) is exact for the quotients here (< 2^52)."""
    f = math.floor(x)
    return int(f) + (1 if x - f >= 0.5 else 0)


def ratio(shape, lane_weights, absent_weight, requested, capacity):
    """requested / capacity: lane -> value, a missing key counting 0."""
    node_score = weight_sum = 0
    for d, w in enumerate(lane_weights):
        if w == 0:
            continue
        s = broken_linear(shape, utilization(requested.get(d, 0), capacity.get(d, 0)))
        if s > 0:
            node_score += s * w
            weight_sum += w
    if absent_weight:   # every node has capacity 0 of these resources
        s = broken_linear(shape, utilization(0, 0))
        if s > 0:
            node_score += s * absent_weight
            weight_sum += absent_weight
    if weight_sum == 0:
        return 0
    return go_round(node_score / weight_sum)   # int / int is the correctly rounded binary64 quotient, as in Go


def pair_ratio(setting, node, node_nz_i, pod_nz_p, req):
    """Ratio of a pod (request `req`, non-zero pair pod_nz_p) on a node (live Node object, non-zero pair node_nz_i)."""
    _, shape, lane_weights, absent_weight = (tuple(setting) + (0,))[:4]
    requested = {0: node_nz_i[0] + pod_nz_p[0], 1: node_nz_i[1] + pod_nz_p[1],
                 2: i64(node.req.EphemeralStorage + req.EphemeralStorage)}
    capacity = {0: node.alloc.MilliCPU, 1: node.alloc.Memory, 2: node.alloc.EphemeralStorage}
    for d in range(4, len(lane_weights)):
        requested[d] = i64(node.req.ScalarResources.get(d, 0) + req.ScalarResources.get(d, 0))
        capacity[d] = node.alloc.ScalarResources.get(d, 0)
    return ratio(shape, lane_weights, absent_weight, requested, capacity)


def total(setting, weights, node, node_nz_i, pod_nz_p, req):
    s = priority_score(node_nz_i[0] + pod_nz_p[0], node.alloc.MilliCPU, node_nz_i[1] + pod_nz_p[1], node.alloc.Memory,
                       weights)
    if setting[0] == 0:
        return s
    return i64(s + setting[0] * pair_ratio(setting, node, node_nz_i, pod_nz_p, req))


def priority_rows(snap, node_nz, pod_nz, K, setting, weights=(1, 0, 1)):
    """Per pod: [(node, score), ...] of its fitting nodes, score descending then node ascending, padded to K with
    (-1, INT64_MIN).  setting = (weight, shape, lane_weights[, absent_weight])."""
    nt, pt = snap.nodes, snap.pods
    nodes = [Node(nt, i) for i in range(nt.n)]
    aff_bits = getattr(snap, "aff_bits", None)
    out = []
    for p in range(pt.n):
        req = resource_from(pt.req[:, p], int(pt.req_present[p]), nt.lanes)
        pnz = (int(pod_nz[0][p]), int(pod_nz[1][p]))
        cand = []
        for i, node in enumerate(nodes):
            if fits(node, pt, p, i, aff_bits, nt.lanes):
                cand.append((total(setting, weights, node, (int(node_nz[0][i]), int(node_nz[1][i])), pnz, req), i))
        cand.sort(key=lambda t: (-t[0], t[1]))
        row = [(i, s) for s, i in cand[:K]]
        out.append(row + [(-1, INT64_MIN)] * (K - len(row)))
    return out


class RatioChooser(PriorityChooser):
    """PriorityChooser's node choice with the ratio term on the live nodes (their requested and keys grow with every
    assume) and the live non-zero column."""

    def __init__(self, node_nz, pod_nz, weights, setting):
        super().__init__(node_nz, pod_nz, weights)
        self.setting = setting

    def __call__(self, nodes, pt, p, req):
        from pyref import check_fit, compare_resource_and_require, single_node_resource
        sel, tol = int(pt.sel_mask[p]), int(pt.tol_mask[p])
        req_full = resource_from(pt.req[:, p], int(pt.req_present[p]), len(self.setting[2]))
        pnz = (int(self.pod_nz[0][p]), int(self.pod_nz[1][p]))
        best, best_s = -1, None
        for i, node in enumerate(nodes):
            if (node.flags & 0x0F) or not check_fit(sel, tol, node):
                continue
            if not compare_resource_and_require(single_node_resource(node, sel, tol, 1.0), req):
                continue
            s = total(self.setting, self.weights, node, (self.node_nz[0][i], self.node_nz[1][i]), pnz, req_full)
            if best < 0 or s > best_s:
                best, best_s = i, s
        return best
