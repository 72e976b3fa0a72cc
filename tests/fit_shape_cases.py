"""Designed rounds for every instantiated gang_fit lane shape (LW wide, LN narrow, LS scaled lanes), and pairs of tables
on both sides of each limit of the lane classifier.

classify() restates the classifier's rule (classify_lanes in engine.cu) from the rule itself:

  narrow  max |alloc| and max |requested| over every node (and, on the pods lane, max |pod_count|) <= NODE_LIMIT, and
          max |request| over every pod, with or without the key, <= POD_LIMIT;
  scaled  otherwise, when every residual int64(float32(alloc) * 1.0) - used of a node that holds the key (used: the
          pods lane's pod_count when its requested value is 0) and every pod's request is a multiple of 2^k, where k is
          the smallest unit with max |value| >> k <= SCALED_LIMIT;
  wide    otherwise.
  Then: at most FIT_MAX_LN narrow lanes (the top scalar lanes go wide first); scaled lanes go back to wide, last first,
  until (LW, LN, LS) is a shape the variant table holds; and every lane is wide when no fixed lane is narrow or the
  shape still does not exist.

The constants are read from the sources.  SHAPE_CASES gives, for each shape, the value design of every lane ("n"
narrow, "w" wide, a number k: scaled in units of 2^k); build() turns a design into a snapshot in which:

  - node n sits at level n % 3 on every lane: residual base + level x unit;
  - for every lane one pod asks exactly the level-1 residual, so the pairs differ by -1, 0 and +1 unit on that lane;
  - for every scaled lane one pod sits C - 1, C and C + 1 units below the residuals (C the clamp 2^(27-k), or 1 above
    unit 27), and for every wide lane two pods leave 2^31 + 6..8 (high word 0, low word >= 2^31) and 2^32 + 2..4;
  - on every lane a pod does not decide on, a narrow lane is asked -(2^26 - 1); one pod decides on none: those
    pods' narrow minimum reaches 2^27 - 3, so the packed best-node key comes close to 2^31;
  - every best score is reached by every node of one level: ties in every tile (and every tail piece) that only the
    lowest node index breaks;
  - on each scalar lane one node in sixteen lacks the key (alloc key only, requested key only, or neither) and the pods
    that do not decide on it either lack it, ask for it, or ask 0 of it.

Shapes with no narrow lane are the all-wide fallback: from L = 6 up a fixed lane is narrow but more than four lanes are
not (a shape the table does not hold; L = 16 is sixteen narrow lanes capped to (8, 8, 0)), for L = 4 and 5 no fixed
lane is narrow.

BORDERS are pairs of tables a limit tells apart; EXPECTED_BORDERS records what classify() gives for each side."""
from __future__ import annotations

import os
import re

import numpy as np

from randsnap import S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _src(*path):
    with open(os.path.join(ROOT, *path)) as f:
        return f.read()


COMMON = _src("batch-scheduler_b200", "csrc", "common.cuh")
FIT = _src("batch-scheduler_b200", "csrc", "fit.cuh")
FIT_CAP_LOG2 = int(re.search(r"constexpr int FIT_CAP_LOG2 = (\d+);", COMMON).group(1))
SCALED_LIMIT = 1 << int(re.search(r"constexpr int64_t SCALED_LIMIT = \(int64_t\)1 << (\d+);", COMMON).group(1))
FIT_MAX_LN = int(re.search(r"constexpr int FIT_MAX_LN = (\d+);", FIT).group(1))
FIT_WS_COMBOS = tuple((int(a), int(b)) for a, b in re.findall(
    r"\{(\d+), (\d+)\}", re.search(r"FIT_WS_COMBOS\[\] = \{(.*)\};", FIT).group(1)))
MAX_LANES = int(re.search(r"#define BS_MAX_LANES (\d+)", _src("include", "bsched.h")).group(1))
# a narrow request |q| <= POD_LIMIT against |float32(alloc)| + |used| <= 2 NODE_LIMIT + 1: every narrow difference stays
# below 2^FIT_CAP_LOG2, so a fitting pair's score and the node's word index share one 31-bit key
POD_LIMIT = (1 << (FIT_CAP_LOG2 - 1)) - 1
NODE_LIMIT = POD_LIMIT >> 1
VALUE_LIMIT = 1 << int(re.search(r"#define BS_VALUE_LIMIT \(\(int64_t\)1 << (\d+)\)", _src("include", "bsched.h")).group(1))
WIDE, NARROW, SCALED = 0, 1, 2
I64_MIN = np.iinfo(np.int64).min
I64_MAX = np.iinfo(np.int64).max


def variant_exists(lw, ln, ls):
    if ln == 0:
        return ls == 0 and 4 <= lw <= MAX_LANES
    return ln <= FIT_MAX_LN and 4 <= lw + ln + ls <= MAX_LANES and (lw, ls) in FIT_WS_COMBOS


def instantiated_shapes():
    """Every (LW, LN, LS) the variant table holds."""
    out = [(lw, 0, 0) for lw in range(4, MAX_LANES + 1)]
    out += [(lw, ln, ls) for ln in range(1, FIT_MAX_LN + 1) for lw, ls in FIT_WS_COMBOS if variant_exists(lw, ln, ls)]
    return out


def clamp_units(k):
    """C: a scaled difference of C or more units (2^k each) cannot be a fitting pair's minimum."""
    return 1 << (FIT_CAP_LOG2 - k) if k <= FIT_CAP_LOG2 else 1


# ---- the restatement -------------------------------------------------------------------------------------------

def f32(a):
    """int64(float32(a)) element-wise, float32 rounding to nearest even done once (numpy goes through float64, which
    rounds first above 2^53)."""
    a = np.asarray(a, np.int64)
    out = a.astype(np.float64).astype(np.float32).astype(np.int64)
    for i in np.flatnonzero(np.abs(a) > (1 << 53)):
        v = int(a[i])
        m, sh = abs(v), abs(v).bit_length() - 24
        q, r = m >> sh, m & ((1 << sh) - 1)
        half = 1 << (sh - 1)
        q += r > half or (r == half and q & 1)
        out[i] = (q << sh) * (1 if v > 0 else -1)
    return out


def _absmax(a):
    return int(np.abs(np.asarray(a, np.int64)).max()) if np.size(a) else 0


def _or(a):
    return int(np.bitwise_or.reduce(np.asarray(a, np.int64).view(np.uint64))) if np.size(a) else 0


def _ctz(v):
    return (v & -v).bit_length() - 1 if v else 63


def node_residuals(nt, d):
    """Residuals at percent 1.0 of the nodes that hold lane d's key (the fixed lanes: every node)."""
    used = nt.requested[d]
    if d == S.LANE_PODS:
        used = np.where(used == 0, nt.pod_count.astype(np.int64), used)
    left = f32(nt.alloc[d]) - used
    if d >= 4:
        left = left[(((nt.alloc_present & nt.req_present) >> np.uint32(d)) & np.uint32(1)).astype(bool)]
    return left


def classify(nodes, pods, history=()):
    """(kind [L] uint8, unit [L] uint8) of the fit kernel for these tables.  history: node tables whose rows were
    uploaded earlier and later replaced by row updates (the statistics only widen)."""
    tables = [nodes, *history]
    L = nodes.lanes
    kind, unit = np.zeros(L, np.uint8), np.zeros(L, np.uint8)
    for d in range(L):
        used = max(_absmax(t.requested[d]) for t in tables)
        if d == S.LANE_PODS:
            used = max(used, max(_absmax(t.pod_count) for t in tables))
        alloc = max(_absmax(t.alloc[d]) for t in tables)
        req = _absmax(pods.req[d])
        if alloc <= NODE_LIMIT and used <= NODE_LIMIT and req <= POD_LIMIT:
            kind[d] = NARROW
            continue
        left = [node_residuals(t, d) for t in tables]
        mx = max([req] + [_absmax(x) for x in left])
        k_avail = min([_ctz(_or(pods.req[d]))] + [_ctz(_or(x)) for x in left])
        k_need = 0
        while k_need < 63 and (mx >> k_need) > SCALED_LIMIT:
            k_need += 1
        if k_need <= k_avail:
            kind[d], unit[d] = SCALED, k_need
    fixed_narrow = (kind[:4] == NARROW).any()
    for d in range(L - 1, 3, -1):
        if fixed_narrow and (kind == NARROW).sum() > FIT_MAX_LN and kind[d] == NARROW:
            kind[d] = WIDE
    for d in range(L - 1, -1, -1):
        if fixed_narrow and not variant_exists(*shape_of(kind)) and kind[d] == SCALED:
            kind[d], unit[d] = WIDE, 0
    if not fixed_narrow or not variant_exists(*shape_of(kind)):
        kind[:], unit[:] = WIDE, 0
    return kind, unit


def shape_of(kind):
    kind = np.asarray(kind)
    return int((kind == WIDE).sum()), int((kind == NARROW).sum()), int((kind == SCALED).sum())


def lane_tokens(kind, unit):
    """"n w s13 ..." for a lane map."""
    return " ".join("n" if k == NARROW else f"s{u}" if k == SCALED else "w" for k, u in zip(kind, unit))


# ---- designed snapshots ----------------------------------------------------------------------------------------

# (LW, LN, LS) -> the value design of lanes 0..L-1: "n" narrow, "w" wide, k scaled in units of 2^k.  The classes move
# round the lanes from one shape to the next, and the scaled units run through 0, 13, 27, 28, 5, 20, 1, 26, 9.
SHAPE_CASES = {
    (4, 0, 0): "w 0 w 27",
    (5, 0, 0): "13 w w w n",
    (6, 0, 0): "w w n 1 w w",
    (7, 0, 0): "26 w w n w w n",
    (8, 0, 0): "n 9 w w w n w n",
    (9, 0, 0): "w n 0 w w w w w w",
    (10, 0, 0): "w w n 13 w w w w w n",
    (11, 0, 0): "27 w w n w w w w n w n",
    (12, 0, 0): "n 28 w w w w w w w w w w",
    (13, 0, 0): "w n 5 w w w w w w w w w n",
    (14, 0, 0): "w w n 20 w w w w w w w n w n",
    (15, 0, 0): "1 w w n w w w w w w w w w w w",
    (16, 0, 0): "n n n n n n n n n n n n n n n n",
    (3, 1, 0): "w n w w",
    (4, 1, 0): "n w w w w",
    (0, 1, 3): "0 13 27 n",
    (1, 1, 2): "n 28 5 w",
    (2, 1, 1): "w n 20 w",
    (2, 2, 0): "w w n n",
    (3, 2, 0): "n n w w w",
    (4, 2, 0): "n w w w w n",
    (0, 2, 2): "26 n n 1",
    (0, 2, 3): "n n 9 0 13",
    (1, 2, 1): "n 27 w n",
    (1, 2, 2): "n n 28 5 w",
    (2, 2, 1): "n n 20 w w",
    (1, 3, 0): "n w n n",
    (2, 3, 0): "n n n w w",
    (3, 3, 0): "w w n n n w",
    (4, 3, 0): "n w w w w n n",
    (0, 3, 1): "n 1 n n",
    (0, 3, 2): "n n n 26 9",
    (0, 3, 3): "n 0 13 27 n n",
    (1, 3, 1): "n n n 28 w",
    (1, 3, 2): "20 w n n n 5",
    (2, 3, 1): "w n n n 1 w",
    (0, 4, 0): "n n n n",
    (1, 4, 0): "n n n n w",
    (2, 4, 0): "n n w w n n",
    (3, 4, 0): "n n n w w w n",
    (4, 4, 0): "n n n n w w w w",
    (0, 4, 1): "n n n n 26",
    (0, 4, 2): "n n n n 9 0",
    (0, 4, 3): "n n 13 27 28 n n",
    (1, 4, 1): "n n 5 w n n",
    (1, 4, 2): "w n n n n 20 1",
    (2, 4, 1): "n n n 26 w w n",
    (0, 5, 0): "n n n n n",
    (1, 5, 0): "n n n n n w",
    (2, 5, 0): "n n n n n w w",
    (3, 5, 0): "w w n n n n n w",
    (4, 5, 0): "w w w n n n n n w",
    (0, 5, 1): "n 9 n n n n",
    (0, 5, 2): "n n n n 0 13 n",
    (0, 5, 3): "n n n 27 28 5 n n",
    (1, 5, 1): "20 w n n n n n",
    (1, 5, 2): "n n n n n 1 26 w",
    (2, 5, 1): "n n 9 w w n n n",
    (0, 6, 0): "n n n n n n",
    (1, 6, 0): "w n n n n n n",
    (2, 6, 0): "n n w w n n n n",
    (3, 6, 0): "n n n n n w w w n",
    (4, 6, 0): "n n n n n n w w w w",
    (0, 6, 1): "n n n n n n 0",
    (0, 6, 2): "n n n n n n 13 27",
    (0, 6, 3): "20 n n n n n n 28 5",
    (1, 6, 1): "1 w n n n n n n",
    (1, 6, 2): "9 w n n n n n n 26",
    (2, 6, 1): "n n n n 0 w w n n",
    (0, 7, 0): "n n n n n n n",
    (1, 7, 0): "n n n n n w n n",
    (2, 7, 0): "n n w w n n n n n",
    (3, 7, 0): "n n n n n n n w w w",
    (4, 7, 0): "w w n n n n n n n w w",
    (0, 7, 1): "n 13 n n n n n n",
    (0, 7, 2): "n n n n 27 28 n n n",
    (0, 7, 3): "n n n n n n n 5 20 1",
    (1, 7, 1): "n n n n n 26 w n n",
    (1, 7, 2): "n n n n n n n 9 0 w",
    (2, 7, 1): "n n 13 w w n n n n n",
    (0, 8, 0): "n n n n n n n n",
    (1, 8, 0): "n n n n n n n n w",
    (2, 8, 0): "n n n n n n n n w w",
    (3, 8, 0): "n n n n n w w w n n n",
    (4, 8, 0): "n n n n n n n n w w w w",
    (0, 8, 1): "n 27 n n n n n n n",
    (0, 8, 2): "n n n n n n n n 28 5",
    (0, 8, 3): "n n n 20 1 26 n n n n n",
    (1, 8, 1): "n n n n n n n n 9 w",
    (1, 8, 2): "n n 0 13 w n n n n n n",
    (2, 8, 1): "n n n n n n n 27 w w n",

}

WIDE_BASE = (1 << 33) + 1   # odd wide residuals: no power-of-two unit


def parse_layout(layout):
    return [t if t in ("n", "w") else int(t) for t in layout.split()]


def lane_design(tok, level):
    """(alloc, requested) of a node at `level` on a lane of design `tok`, and the level-1 residual and the unit."""
    lv = np.asarray(level, np.int64)
    if tok == "n":      # float32(2^25 - 1) = 2^25: residuals 2^26 - 4 + level, |requested| <= NODE_LIMIT
        return np.full(lv.shape, NODE_LIMIT), -(NODE_LIMIT - 3) - lv, (1 << 26) - 3, 1
    if tok == "w":
        return np.full(lv.shape, 1 << 34), (1 << 34) - WIDE_BASE - lv, WIDE_BASE + 1, 1
    k = tok             # residuals 2^(29+k) - (2 - level) 2^k: the largest is exactly SCALED_LIMIT units of 2^k
    u = 1 << k
    if (SCALED_LIMIT << k) > VALUE_LIMIT:
        # requests stop at 2^56: residuals 2^56 - (2 - level) 2^k; anchor_nodes() hold the magnitude that needs unit k
        return np.full(lv.shape, VALUE_LIMIT), (2 - lv) * u, VALUE_LIMIT - u, u
    return np.full(lv.shape, SCALED_LIMIT << (k - 1) if k else SCALED_LIMIT >> 1), \
        -(SCALED_LIMIT << (k - 1) if k else SCALED_LIMIT >> 1) + (2 - lv) * u, (SCALED_LIMIT << k) - u, u


def anchor_nodes(N):
    """Nodes whose residual on a lane of unit k > 27 is 2^57 - (2 - level) 2^k (alloc 2^56, requested -2^56 + ...)."""
    return np.arange(N) % 7 == 5


def generous(tok):
    """A request that leaves any node far more than any decisive difference."""
    return -POD_LIMIT if tok == "n" else 1 if tok == "w" else 1 << tok


def build(layout, N, name, copies=2, G=4):
    lay = parse_layout(layout) if isinstance(layout, str) else list(layout)
    L = len(lay)
    nt = S.NodeTable.empty(N, L)
    level = np.arange(N) % 3
    for d, tok in enumerate(lay):
        nt.alloc[d], nt.requested[d], _, _ = lane_design(tok, level)
        if tok not in ("n", "w") and (SCALED_LIMIT << tok) > VALUE_LIMIT:
            nt.requested[d, anchor_nodes(N)] -= VALUE_LIMIT
        if d >= 4:
            # one node in sixteen lacks the key: alloc key only, requested key only, or neither
            absent = (np.arange(N) // 3) % MAX_LANES == d     # a node lacks one key at most
            how = (np.arange(N) // (3 * MAX_LANES)) % 3
            bit = np.uint32(1 << d)
            nt.alloc_present |= np.where(absent & (how != 0), np.uint32(0), bit)
            nt.req_present |= np.where(absent & (how != 1), np.uint32(0), bit)
    # (deciding lane, request on it, whether the narrow minimum stays near 2^27: no narrow lane asked 0)
    roles = [(-1, 0, True), (-2, 0, False)]                     # no deciding lane; -2: asks 0 of every scalar key
    for d, tok in enumerate(lay):
        _, _, l1, u = lane_design(tok, 1)
        roles.append((d, l1, False))                            # -1, 0, +1 unit
        if tok not in ("n", "w"):
            roles.append((d, l1 - clamp_units(tok) * u, True))  # C - 1, C, C + 1 units
        if tok == "w":
            roles += [(d, l1 - (1 << 31) - 7, True), (d, l1 - (1 << 32) - 3, True)]
    P = len(roles) * copies
    pt = S.PodTable.empty(P, L)
    for c in range(copies):
        for i, (dd, q, high) in enumerate(roles):
            p = c * len(roles) + i
            for d, tok in enumerate(lay):
                if d == dd:
                    pt.req[d, p] = q
                    pt.req_present[p] |= np.uint32(1 << d) if d >= 4 else 0
                    continue
                mode = 1 if d < 4 else 2 if dd == -2 else (p + d + c) % (2 if high and tok == "n" else 3)
                pt.req[d, p] = 0 if mode == 2 else generous(tok)   # mode 0: no key (the value still counts)
                if mode:
                    pt.req_present[p] |= np.uint32(1 << d) if d >= 4 else 0
    pt.gid = (np.arange(P) % G).astype(np.int32)
    pt.ts_ns = 1_700_000_000 * 10**9 + np.arange(P, dtype=np.int64) * 1000
    gt = S.GroupTable.empty(G, L)
    gt.min_member[:] = 1
    gt.flags[:] = S.GROUP_HAS_POD | S.GROUP_HAS_MINRES
    gt.creation_ns = 1_600_000_000 * 10**9 + np.arange(G, dtype=np.int64)
    gt.name_rank = np.arange(G, dtype=np.uint32)
    return S.Snapshot(nt, pt, gt, name)


SIZES = {"full": 1000, "split": 1100}   # N: one bitmap line (full-range units) / two (tail units cut into pieces)


def shape_snapshot(shape, size):
    return build(SHAPE_CASES[shape], SIZES[size], "shape{}-{}-{}_{}".format(*shape, size))


# ---- border pairs ----------------------------------------------------------------------------------------------

BORDER_BASE = "n w 13 n n"   # (1, 3, 1); lane 4 is a narrow scalar lane, lane 2 scaled in units of 2^13
BORDER_N = 300


def _base(layout=BORDER_BASE, name="border"):
    return build(layout, BORDER_N, name, copies=1)


def border_pair(name):
    """The two tables of border case `name`: (inside, outside)."""
    def pair(edit, a, b, layout=BORDER_BASE):
        out = []
        for side, v in (("in", a), ("out", b)):
            s = _base(layout, f"{name}_{side}")
            edit(s, v)
            out.append(s)
        return tuple(out)

    if name.startswith(("alloc", "requested")):
        col, sign = name.split("_")
        s = 1 if sign == "pos" else -1
        return pair(lambda sn, v: getattr(sn.nodes, col).__setitem__((4, 7), v), s * NODE_LIMIT, s * (NODE_LIMIT + 1))
    if name.startswith("pod_count"):
        s = 1 if name.endswith("pos") else -1
        return pair(lambda sn, v: sn.nodes.pod_count.__setitem__(7, v), s * NODE_LIMIT, s * (NODE_LIMIT + 1),
                    layout="w w 13 n n")
    if name.startswith("pod_req"):
        s = 1 if name.endswith("pos") else -1
        return pair(lambda sn, v: sn.pods.req.__setitem__((4, 3), v), s * POD_LIMIT, s * (POD_LIMIT + 1))
    if name == "pods_lane_pod_count":
        # requested 0 on the pods lane: the residual is alloc - pod_count
        def edit(sn, v):
            sn.nodes.requested[3, 7] = 0
            sn.nodes.pod_count[7] = v
        return pair(edit, 1 << 13, (1 << 13) + 1, layout="n w w 13 n")
    if name.startswith("scaled_limit"):
        top = SCALED_LIMIT << 13
        if name.endswith("node"):     # node 2 (level 2) already sits at exactly SCALED_LIMIT units
            return pair(lambda sn, v: sn.nodes.requested.__setitem__((2, 2), sn.nodes.alloc[2, 2] - v), top,
                        top + (1 << 13))
        s = 1 if name.endswith("pos") else -1
        return pair(lambda sn, v: sn.pods.req.__setitem__((2, 0), v), s * top, s * (top + (1 << 13)))
    if name == "odd_node":
        return pair(lambda sn, v: sn.nodes.requested.__setitem__((2, 7), sn.nodes.requested[2, 7] + v), 1 << 13, 1)
    if name == "odd_pod":
        return pair(lambda sn, v: sn.pods.req.__setitem__((2, 4), v), 3 << 13, (3 << 13) + 1)
    if name == "odd_node_without_key":
        # node 7 lacks lane 5's key (inside) or holds it (outside); its residual there is odd
        def edit(sn, v):
            sn.nodes.requested[5, 7] += 1
            sn.nodes.alloc_present[7] = (sn.nodes.alloc_present[7] & ~np.uint32(1 << 5)) | np.uint32(v << 5)
            sn.nodes.req_present[7] |= np.uint32(1 << 5)
        return pair(edit, 0, 1, layout="n w w n n 13")
    if name == "pod_without_key_huge":
        def edit(sn, v):
            sn.pods.req_present[5] &= ~np.uint32(1 << 4)
            sn.pods.req[4, 5] = v
        return pair(edit, 1 << 20, 1 << 40)
    if name == "float32_rounding":
        # lane 4 residuals 2^30 and requests 2: unit 1, unless node 7's alloc keeps an odd value through float32
        def edit(sn, v):
            sn.nodes.alloc[4] = 1 << 30
            sn.nodes.requested[4] = 0
            sn.nodes.alloc[4, 7] = v
            sn.pods.req[4] = 2
        return pair(edit, (1 << 24) + 1, (1 << 24) - 1, layout="n w 13 n w")
    if name == "narrow_cap":
        return _base(" ".join(["n"] * 8), f"{name}_in"), _base(" ".join(["n"] * 9), f"{name}_out")
    if name == "sixteen_narrow":
        return _base(" ".join(["n"] * 12), f"{name}_in"), _base(" ".join(["n"] * 16), f"{name}_out")
    if name == "missing_combo":
        return _base("n 13 w w", f"{name}_in"), _base("n 13 w w w", f"{name}_out")
    if name == "missing_combo_walk":
        return _base("n 0 13 27", f"{name}_in"), _base("n 0 13 27 28", f"{name}_out")
    if name == "no_fixed_narrow":
        return _base("n w w w n", f"{name}_in"), _base("w w w w n", f"{name}_out")
    raise KeyError(name)


# name -> (lane map inside, lane map outside), as classify() gives them
EXPECTED_BORDERS = {
    "alloc_pos": ("n w s13 n n", "n w s13 n s0"),
    "alloc_neg": ("n w s13 n n", "n w s13 n s0"),
    "requested_pos": ("n w s13 n n", "n w s13 n s0"),
    "requested_neg": ("n w s13 n n", "n w s13 n s0"),
    "pod_count_pos": ("w w s13 n n", "w w w w w"),
    "pod_count_neg": ("w w s13 n n", "w w w w w"),
    "pod_req_pos": ("n w s13 n n", "n w s13 n s0"),
    "pod_req_neg": ("n w s13 n n", "n w s13 n s0"),
    "pods_lane_pod_count": ("n w w s13 n", "n w w w n"),
    "scaled_limit_node": ("n w s13 n n", "n w w n n"),
    "scaled_limit_pos": ("n w s13 n n", "n w w n n"),
    "scaled_limit_neg": ("n w s13 n n", "n w w n n"),
    "odd_node": ("n w s13 n n", "n w w n n"),
    "odd_pod": ("n w s13 n n", "n w w n n"),
    "odd_node_without_key": ("n w w n n s13", "n w w n n w"),
    "pod_without_key_huge": ("n w s13 n n", "n w s13 n w"),
    "float32_rounding": ("n w s13 n s1", "n w s13 n w"),
    "narrow_cap": ("n n n n n n n n", "n n n n n n n n w"),
    "sixteen_narrow": ("n n n n n n n n w w w w", "w w w w w w w w w w w w w w w w"),
    "missing_combo": ("n s13 w w", "n w w w w"),
    "missing_combo_walk": ("n s0 s13 s27", "n w w w w"),
    "no_fixed_narrow": ("n w w w n", "w w w w w"),
}
BORDERS = tuple(EXPECTED_BORDERS)


# ---- what decides each pair ------------------------------------------------------------------------------------

def lane_differences(oracle, snap):
    """(diff [L, P, N] int64 with I64_MAX where the lane is not compared, class_ok [P, N]): left - request per lane
    from the oracle's residuals; class_ok is False where the pod asks a non-zero amount of a key the node lacks."""
    nt, pt = snap.nodes, snap.pods
    left, lpres = oracle.node_left(nt, 0, 0, 1.0)
    L = nt.lanes
    bits = (1 << np.arange(L, dtype=np.uint32)).astype(np.uint32)
    both = ((lpres[None, :] & pt.req_present[:, None])[None] & bits[:, None, None]) != 0
    both[:4] = True
    diff = np.where(both, left[:, None, :] - pt.req[:, :, None], I64_MAX)
    nz = np.zeros(pt.n, np.uint32)
    for d in range(4, L):
        nz |= np.where(((pt.req_present >> np.uint32(d)) & 1).astype(bool) & (pt.req[d] != 0), np.uint32(1 << d), 0
                       ).astype(np.uint32)
    class_ok = (nz[:, None] & ~lpres[None, :]) == 0
    return diff, class_ok
