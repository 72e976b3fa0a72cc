"""A second, independent restatement of the ImageLocality and NodePreferAvoidPods priorities (include/bsched.h
bs_set_locality_weights) in pure Python over the Go-like objects of tests/pyref.py, written from kube-scheduler
v1.17's image_locality.go and node_prefer_avoid_pods.go [upstream, from memory] without looking at the C
restatement.  The resource part of the score is tests/pyref_ratio_priority.py's, the node priorities' part
tests/pyref_node_priority.py's.  Python floats are IEEE binary64 with round to nearest, as Go's float64; Python ints
are masked to int64 where Go would wrap."""
from pyref import Node, i64, resource_from
from pyref_node_priority import affinity_count, normalize_reduce, taint_count
from pyref_priority import INT64_MIN, fits
from pyref_ratio_priority import RatioChooser, total

IMAGE_NONE = 0xFFFFFFFF
AVOID_NONE = 0xFF
MB = 1024 * 1024
MIN_THRESHOLD = 23 * MB
MAX_THRESHOLD = 1000 * MB


def normalized_image_name(name: str) -> str:
    """normalizedImageName: a name without a tag gets ":latest" (a ':' before the last '/' is a registry port)."""
    if name.rfind(":") <= name.rfind("/"):
        name = name + ":latest"
    return name


def reported(image_bits, i, n):
    return (int(image_bits[i][n // 32]) >> (n % 32)) & 1


def image_states(image_size, image_bits, n_nodes):
    """[(size, NumNodes)] per name: the nodes of the snapshot that report it."""
    return [(int(image_size[i]), sum(reported(image_bits, i, n) for n in range(n_nodes)))
            for i in range(len(image_size))]


def scaled_image_score(size, num_nodes, total_num_nodes):
    """scaledImageScore: int64(float64(size) * (float64(NumNodes) / float64(totalNumNodes)))."""
    spread = float(num_nodes) / float(total_num_nodes)
    return int(float(size) * spread)   # int() truncates toward zero


def calculate_priority(sum_scores):
    """calculatePriority (v1.17: one fixed upper threshold, not scaled by the number of containers)."""
    sum_scores = min(max(sum_scores, MIN_THRESHOLD), MAX_THRESHOLD)
    return 100 * (sum_scores - MIN_THRESHOLD) // (MAX_THRESHOLD - MIN_THRESHOLD)


def image_locality(states, image_bits, ids, n, n_nodes):
    """ImageLocality of the pod whose containers name `ids` (dictionary ids, repeats kept) on node n."""
    s = 0
    for i in ids:
        if reported(image_bits, i, n):
            s += scaled_image_score(states[i][0], states[i][1], n_nodes)
    return calculate_priority(s)


def prefer_avoid_pods(avoid_mask_n, bit):
    """NodePreferAvoidPods: 0 when the node's annotation lists the pod's RC / RS controller, else 100."""
    if int(bit) == AVOID_NONE:
        return 100
    return 0 if (int(avoid_mask_n) >> int(bit)) & 1 else 100


def pod_ids(cls, off, ids):
    if int(cls) == IMAGE_NONE:
        return []
    return [int(x) for x in ids[int(off[int(cls)]):int(off[int(cls) + 1])]]


def priority_rows(snap, node_nz, pod_nz, K, loc, lw, setting=(0, ((0, 100), (100, 0)), [0] * 4), weights=(1, 0, 1),
                  prefs=None, pw=(0, 0), pods=None):
    """Per pod: [(node, score), ...] of its fitting nodes, score descending then node ascending, padded to K with
    (-1, INT64_MIN).  loc = ((image_size, image_bits, avoid_mask), (image_class, class_offset, class_images,
    avoid_bit)), lw = (ImageLocality, NodePreferAvoidPods) weights; prefs / pw: the node priorities (None: off)."""
    nt, pt = snap.nodes, snap.pods
    (size, bits, avoid), (cls, off, ids, abit) = loc
    w_img, w_avoid = lw
    if len(setting[2]) != nt.lanes:
        setting = (setting[0], setting[1], list(setting[2]) + [0] * (nt.lanes - len(setting[2]))) + tuple(setting[3:])
    states = image_states(size, bits, nt.n)
    nodes = [Node(nt, i) for i in range(nt.n)]
    aff_bits = getattr(snap, "aff_bits", None)
    out = []
    for p in (range(pt.n) if pods is None else pods):
        fit = [i for i in range(nt.n) if fits(nodes[i], pt, p, i, aff_bits, nt.lanes)]
        if prefs is not None and any(pw):
            taints, table, tol, pcls = prefs
            tt = normalize_reduce({i: taint_count(taints[i], tol[p]) for i in fit}, True)
            na = normalize_reduce({i: affinity_count(table, pcls[p], i) for i in fit}, False)
        req = resource_from(pt.req[:, p], int(pt.req_present[p]), nt.lanes)
        pnz = (int(pod_nz[0][p]), int(pod_nz[1][p]))
        mine = pod_ids(cls[p], off, ids)
        cand = []
        for i in fit:
            s = total(setting, weights, nodes[i], (int(node_nz[0][i]), int(node_nz[1][i])), pnz, req)
            if prefs is not None and any(pw):
                s += pw[0] * tt[i] + pw[1] * na[i]
            if w_img:
                s += w_img * image_locality(states, bits, mine, i, nt.n)
            s += w_avoid * (prefer_avoid_pods(avoid[i], abit[p]) if w_avoid else 100)
            cand.append((i64(s), i))
        cand.sort(key=lambda t: (-t[0], t[1]))
        row = [(i, s) for s, i in cand[:K]]
        out.append(row + [(-1, INT64_MIN)] * (K - len(row)))
    return out


class LocalityChooser(RatioChooser):
    """tests/pyref_ratio_priority.py's RatioChooser with the two locality terms added per fitting node (static: the
    walk does not change them); for tests/pyref_replay_priority.py's walk."""

    def __init__(self, node_nz, pod_nz, weights, setting, loc, lw, n_nodes):
        super().__init__(node_nz, pod_nz, weights, setting)
        (self.size, self.bits, self.avoid), (self.cls, self.off, self.ids, self.abit) = loc
        self.lw = lw
        self.n_nodes = n_nodes
        self.states = image_states(self.size, self.bits, n_nodes)

    def __call__(self, nodes, pt, p, req):
        from pyref import check_fit, compare_resource_and_require, single_node_resource
        sel, tol = int(pt.sel_mask[p]), int(pt.tol_mask[p])
        req_full = resource_from(pt.req[:, p], int(pt.req_present[p]), len(self.setting[2]))
        pnz = (int(self.pod_nz[0][p]), int(self.pod_nz[1][p]))
        mine = pod_ids(self.cls[p], self.off, self.ids)
        best, best_s = -1, None
        for i, node in enumerate(nodes):
            if (node.flags & 0x0F) or not check_fit(sel, tol, node):
                continue
            if not compare_resource_and_require(single_node_resource(node, sel, tol, 1.0), req):
                continue
            s = total(self.setting, self.weights, node, (self.node_nz[0][i], self.node_nz[1][i]), pnz, req_full)
            if self.lw[0]:
                s += self.lw[0] * image_locality(self.states, self.bits, mine, i, self.n_nodes)
            s = i64(s + self.lw[1] * (prefer_avoid_pods(self.avoid[i], self.abit[p]) if self.lw[1] else 100))
            if best < 0 or s > best_s:
                best, best_s = i, s
        return best
