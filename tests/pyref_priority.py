"""A second, independent restatement of the priority lists (include/bsched.h BS_OUT_PRIORITY) in pure Python over the
Go-like objects of tests/pyref.py, written from kube-scheduler v1.17's resource priorities [upstream, from memory]
without looking at the C restatement.  Python floats are IEEE binary64 like Go's float64; Python ints are masked to
int64 where Go would wrap.  Used to cross-check tests/priority_ref.c on small cases."""
import math

from pyref import M64, Node, check_fit, compare_resource_and_require, i64, resource_from, single_node_resource

INT64_MIN = -(1 << 63)


def _trunc_div(a, b):   # Go's int64 division truncates toward zero
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b >= 0) else -q


def least_requested(requested, capacity):
    if capacity == 0 or requested > capacity:
        return 0
    return _trunc_div((capacity - requested) * 100, capacity)


def most_requested(requested, capacity):
    if capacity == 0 or requested > capacity:
        return 0
    return _trunc_div(requested * 100, capacity)


def fraction_of_capacity(requested, capacity):
    if capacity == 0:
        return 1.0
    return float(requested) / float(capacity)


def balanced(r_cpu, c_cpu, r_mem, c_mem):
    fc, fm = fraction_of_capacity(r_cpu, c_cpu), fraction_of_capacity(r_mem, c_mem)
    if fc >= 1 or fm >= 1:
        return 0
    x = (1 - abs(fc - fm)) * 100.0
    if x < -2.0 ** 63:   # out of int64's range (a negative capacity): the conversion saturates
        return INT64_MIN
    return int(math.trunc(x))


def score(r_cpu, c_cpu, r_mem, c_mem, weights=(1, 0, 1)):
    wl, wm, wb = weights
    least = _trunc_div(least_requested(r_cpu, c_cpu) + least_requested(r_mem, c_mem), 2)
    most = _trunc_div(most_requested(r_cpu, c_cpu) + most_requested(r_mem, c_mem), 2)
    return i64((wl * least + wm * most + wb * balanced(r_cpu, c_cpu, r_mem, c_mem)) & M64)


def fits(node, pt, p, i, aff_bits, L):
    """The pod's Filter verdict on node i as the round computes it: guards, checkFit (and the affinity bit), then
    compareResourceAndRequire against singleNodeResource at percent 1.0."""
    if node.flags & 0x0F:
        return False
    sel, tol = int(pt.sel_mask[p]), int(pt.tol_mask[p])
    if not check_fit(sel, tol, node):
        return False
    aff = 0xFFFFFFFF if getattr(pt, "aff_class", None) is None else int(pt.aff_class[p])
    if aff != 0xFFFFFFFF and not (int(aff_bits[aff, i // 32]) >> (i % 32)) & 1:
        return False
    req = resource_from(pt.req[:, p], int(pt.req_present[p]), L)
    return compare_resource_and_require(single_node_resource(node, sel, tol, 1.0), req)


def priority_rows(snap, node_nz, pod_nz, K, weights=(1, 0, 1)):
    """Per pod: the list of (node, score) of its fitting nodes, score descending then node ascending, padded to K with
    (-1, INT64_MIN)."""
    nt, pt = snap.nodes, snap.pods
    nodes = [Node(nt, i) for i in range(nt.n)]
    aff_bits = getattr(snap, "aff_bits", None)
    out = []
    for p in range(pt.n):
        cand = []
        for i, node in enumerate(nodes):
            if not fits(node, pt, p, i, aff_bits, nt.lanes):
                continue
            r_cpu = int(node_nz[0][i]) + int(pod_nz[0][p])
            r_mem = int(node_nz[1][i]) + int(pod_nz[1][p])
            cand.append((score(r_cpu, node.alloc.MilliCPU, r_mem, node.alloc.Memory, weights), i))
        cand.sort(key=lambda t: (-t[0], t[1]))
        row = [(i, s) for s, i in cand[:K]]
        out.append(row + [(-1, INT64_MIN)] * (K - len(row)))
    return out
