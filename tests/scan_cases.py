"""Node tables whose cluster-scan prefixes follow designed paths, a plain reference of the scan, and a mirror of the
engine's two shortcuts in front of the full scan.

compareClusterResourceAndRequire (core.go:595-632) is true at the first visited prefix whose running sum covers the
need.  The engine decides it in three steps (DESIGN.md §4): per-lane bounds, then the last visited prefix and each
lane's argmax prefix as candidates, then a scan of every visited prefix.  Random snapshots rarely leave a need to the
third step, so the tables here are built from chosen prefix values: a set of targets whose (cpu, memory) values form an
antichain, one peak per lane group elsewhere, and low values everywhere else.  A need equal to a target's prefix is met
there and nowhere else, it passes the bounds, and neither the last prefix nor any argmax prefix meets it; the same need
plus 1 on one lane passes the bounds and is met nowhere.
"""
from __future__ import annotations

import functools
from dataclasses import dataclass, field

import numpy as np

import pyref
from randsnap import S

M64 = (1 << 64) - 1

# node kinds: visited and counted / visited but contributing nothing / skipped by the scan
FIT, TAINTS_ERR, UNFIT_SEL, UNFIT_TOL, NIL, NO_NODE, UNSCHED = range(7)
ZERO_KINDS = (TAINTS_ERR, UNFIT_SEL, UNFIT_TOL)
SKIP_KINDS = (NIL, NO_NODE, UNSCHED)
_FLAGS = {FIT: 0, TAINTS_ERR: S.NODE_TAINTS_ERR, UNFIT_SEL: 0, UNFIT_TOL: 0, NIL: S.NODE_NIL,
          NO_NODE: S.NODE_NO_NODE, UNSCHED: S.NODE_UNSCHEDULABLE}

# the class every trajectory is designed for, and two more that count different node subsets:
# (0, 2) also counts the nodes that fail (1, 0)'s checkFit; (5, 0) drops the fit nodes without label bit 2
SEL, TOL = 0x1, 0x0
CLASSES = [(0x1, 0x0), (0x0, 0x2), (0x5, 0x0)]

LOW = -1000        # default prefix value: LOW - (fit index) on every lane
PEAK = 500


@dataclass
class Table:
    name: str
    snap: object                    # Snapshot with the node table filled, empty pods / groups
    pct: float                      # percent the trajectory is designed at
    targets: list                   # node indices of designed satisfying prefixes
    # designated needs: (need[L] ints, npres, expect "true" / "false", node of the first satisfying prefix or None)
    needs: list = field(default_factory=list)

    @property
    def nodes(self):
        return self.snap.nodes

    @property
    def lanes(self):
        return self.snap.nodes.lanes


def i64(x):
    return pyref.i64(int(x))


# ---------------------------------------------------------------------------------------------------------------
# the plain reference: singleNodeResource and the ordered walk, in Python ints wrapped the way Go's int64 wraps

def node_term(nt, i, sel, tol, pct):
    """(values[L], key mask) of singleNodeResource (core.go:634-670), or None for a node the walk skips."""
    L, f = nt.lanes, int(nt.flags[i])
    if f & 0x07:
        return None
    v = [0] * L
    if f & 0x08 or (int(nt.label_mask[i]) & sel) != sel or (int(nt.taint_mask[i]) & ~tol & M64):
        return v, 0
    pods = int(nt.requested[3, i]) or int(nt.pod_count[i])
    v[3] = i64(pyref.scale(int(nt.alloc[3, i]), pct) - pods)
    for d in range(3):
        v[d] = i64(pyref.scale(int(nt.alloc[d, i]), pct) - int(nt.requested[d, i]))
    keys = 0
    both = int(nt.alloc_present[i]) & int(nt.req_present[i])
    for d in range(4, L):
        if (both >> d) & 1:
            v[d] = i64(pyref.scale(int(nt.alloc[d, i]), pct) - int(nt.requested[d, i]))
            keys |= 1 << d
    return v, keys


def prefixes(nt, sel, tol, pct):
    """Running sums of the walk: pre[L, N] int64 (the value after node i), keys[N] (union of the keys so far),
    visited[N]."""
    L, N = nt.lanes, nt.n
    pre = np.zeros((L, N), np.int64)
    keys = np.zeros(N, np.uint32)
    vis = np.zeros(N, bool)
    run, k = [0] * L, 0
    for i in range(N):
        t = node_term(nt, i, sel, tol, pct)
        if t is not None:
            vis[i] = True
            run = [i64(a + b) for a, b in zip(run, t[0])]
            k |= t[1]
        pre[:, i] = run
        keys[i] = k
    return pre, keys, vis


def satisfied(pre, keys, vis, need, npres):
    """Per node: the walk has visited it and compareResourceAndRequire (core.go:672-699) holds for its prefix."""
    L = pre.shape[0]
    ok = vis.copy()
    for d in range(L):
        if d < 4:
            ok &= pre[d] >= need[d]
        elif (npres >> d) & 1:
            has = ((keys >> np.uint32(d)) & np.uint32(1)).astype(bool)
            ok &= np.where(has, pre[d] >= need[d], need[d] == 0)
    return ok


def first_hit(pre, keys, vis, need, npres):
    """Index of the first satisfying prefix (the walk returns true there), -1 if none."""
    ok = satisfied(pre, keys, vis, need, npres)
    return int(np.argmax(ok)) if ok.any() else -1


@dataclass
class Stats:
    """What the engine folds from its prefix scan (kernels.cuh ClassStats), recomputed from the reference prefixes."""
    maxv: list
    argmax: list
    any_absent: int
    last_visited: int
    unique_max: list


def stats(pre, keys, vis):
    L = pre.shape[0]
    maxv, argmax, unique = [], [], []
    for d in range(L):
        has = vis if d < 4 else vis & ((keys >> np.uint32(d)) & np.uint32(1)).astype(bool)
        if not has.any():
            maxv.append(None), argmax.append(-1), unique.append(True)
            continue
        vals = np.where(has, pre[d], np.iinfo(np.int64).min)
        m = vals.max()
        at = np.flatnonzero(has & (pre[d] == m))
        maxv.append(int(m)), argmax.append(int(at[0])), unique.append(len(at) == 1)
    absent = 0
    for i in np.flatnonzero(vis):
        absent |= ~int(keys[i]) & 0xFFFFFFFF
    last = int(np.flatnonzero(vis)[-1]) if vis.any() else -1
    return Stats(maxv, argmax, absent, last, unique)


BOUNDS, CANDIDATE, STEP3_TRUE, STEP3_FALSE = "bounds", "candidate", "step3-true", "step3-false"


def classify(pre, keys, vis, st, need, npres):
    """Which step decides the need: the per-lane bounds reject it, a candidate prefix (the last visited one or a
    lane's argmax) accepts it, or only the full scan decides, with the given answer."""
    L = pre.shape[0]
    if st.last_visited < 0:
        return BOUNDS
    for d in range(L):
        if d >= 4 and not (npres >> d) & 1:
            continue
        via_present = st.argmax[d] >= 0 and need[d] <= st.maxv[d]
        via_absent = d >= 4 and (st.any_absent >> d) & 1 and need[d] == 0
        if not via_present and not via_absent:
            return BOUNDS
    ok = satisfied(pre, keys, vis, need, npres)
    for c in [st.last_visited] + [a for a in st.argmax if a >= 0]:
        if ok[c]:
            return CANDIDATE
    return STEP3_TRUE if ok.any() else STEP3_FALSE


# ---------------------------------------------------------------------------------------------------------------
# the builder

def build_nodes(L, kinds, P, key_from, pct=1.0, alloc=None, raw=None, seed=0):
    """A node table whose fit nodes' prefixes (class (SEL, TOL)) are P[fit index][lane].

    Scalar lane d's key is carried by the fit nodes at or after key_from[d]; before that the prefix has no key and
    its value is 0 whatever P says.  raw={lane: terms per fit node} gives a lane's terms directly.  With `alloc`
    ([L] per-lane allocatable values, or None for 0), requested = scale(alloc, pct) - term, so the terms go through
    the float32 product at `pct`; with alloc 0 every percent gives the same terms."""
    rng = np.random.default_rng(seed)
    kinds = np.asarray(kinds)
    N = len(kinds)
    nt = S.NodeTable.empty(N, L)
    nt.flags = np.array([_FLAGS[int(k)] for k in kinds], np.uint8)
    nt.label_mask = np.where(kinds == UNFIT_SEL, 0x4, 0x1 | (rng.integers(0, 2, N) << 2)).astype(np.uint64)
    nt.taint_mask = np.where(kinds == UNFIT_TOL, 0x2, 0).astype(np.uint64)
    # nodes that must not count get values that would show if they did
    for i in np.flatnonzero(kinds != FIT):
        nt.alloc[:, i] = rng.integers(1000, 5000, L)
        nt.requested[:, i] = rng.integers(-300, 300, L)
        nt.pod_count[i] = rng.integers(1, 50)
        nt.alloc_present[i] = nt.req_present[i] = ((1 << L) - 1) & ~0xF
    fit = np.flatnonzero(kinds == FIT)
    prev = [0] * L
    for k, i in enumerate(fit):
        cur = [int(x) for x in P[k]]
        for d in range(4, L):
            if i < key_from.get(d, 0):
                cur[d] = 0
        term = [cur[d] - prev[d] for d in range(L)]
        for d, col in (raw or {}).items():
            term[d] = int(col[k])
            cur[d] = i64(prev[d] + term[d])
        prev = cur
        keys = 0
        for d in range(L):
            if d >= 4:
                if i < key_from.get(d, 0):
                    continue
                keys |= 1 << d
            a = 0 if alloc is None else int(alloc[d])
            r = pyref.scale(a, pct) - term[d]
            nt.alloc[d, i] = a
            if d == 3:
                # pods lane: with requested 0 the reference takes the pod count (int32)
                if alloc is None:
                    assert -2**31 <= r < 2**31
                    nt.pod_count[i] = r
                else:
                    nt.requested[3, i] = r
                    nt.pod_count[i] = r       # read only when r == 0
            else:
                assert abs(r) <= 1 << 56, (d, r)
                nt.requested[d, i] = r
        nt.alloc_present[i] = nt.req_present[i] = keys
    return nt


def sprinkle(N, rng, keep, zero=0.06, skip=0.06):
    """Node kinds: mostly FIT, with visited-but-zero and skipped nodes at random positions, never at the indices in
    `keep` or right after them (a zero node there would repeat a designed prefix)."""
    kinds = np.full(N, FIT)
    r = rng.random(N)
    kinds[r < zero] = rng.choice(ZERO_KINDS, N)[r < zero]
    sk = (r >= zero) & (r < zero + skip)
    kinds[sk] = rng.choice(SKIP_KINDS, N)[sk]
    for i in keep:
        kinds[i] = FIT
        j = i + 1
        while j < N and kinds[j] in SKIP_KINDS:
            j += 1
        if j < N:
            kinds[j] = FIT
    return kinds


def antichain(kinds, L, targets, peaks, key_from=None, hi=None, extra=None):
    """P for every fit node: target k gets cpu 100 + 10k, memory 100 + 10(K-1-k), lane d >= 2 the level hi[d];
    peaks[0] tops cpu and every lane >= 2 with memory low, peaks[1] tops memory with the rest low; every other fit
    node LOW - (its fit index).  extra={node: [L] values} overrides single nodes."""
    K = len(targets)
    hi = hi or {d: 50 + d for d in range(2, L)}
    fit = list(np.flatnonzero(np.asarray(kinds) == FIT))
    pos = {i: k for k, i in enumerate(fit)}
    P = [[LOW - k] * L for k in range(len(fit))]
    for k, t in enumerate(targets):
        row = [100 + 10 * k, 100 + 10 * (K - 1 - k)] + [hi[d] for d in range(2, L)]
        P[pos[t]] = row
    a0, a1 = peaks
    P[pos[a0]] = [100 + 10 * K + PEAK, -PEAK] + [hi[d] + PEAK for d in range(2, L)]
    P[pos[a1]] = [-PEAK, 100 + 10 * K + PEAK] + [-PEAK] * (L - 2)
    for i, row in (extra or {}).items():
        P[pos[i]] = list(row)
    return P


def scalar_mask(L):
    return ((1 << L) - 1) & ~0xF


def designated(table, pre, keys, at, npres, bump_lane=None):
    """The need equal to the prefix at node `at` ("true"), and the same need plus 1 on one lane ("false")."""
    need = [int(x) for x in pre[:, at]]
    for d in range(4, table.lanes):
        if (npres >> d) & 1 and not (int(keys[at]) >> d) & 1:
            need[d] = 0            # the prefix has no key d: only a need of 0 is met by it
    d = bump_lane if bump_lane is not None else 0
    plus = list(need)
    plus[d] = i64(plus[d] + 1)
    return [(need, npres, "true", at), (plus, npres, "false", None)]


def _finish(table, designs):
    """Fills table.needs from [(node, npres, bump lane)] against the reference prefixes at the design percent."""
    pre, keys, _ = ref_prefixes(table, SEL, TOL, table.pct)
    for at, npres, lane in designs:
        table.needs += designated(table, pre, keys, at, npres, lane)
    return table


def _snap(nt, name):
    L = nt.lanes
    return S.Snapshot(nt, S.PodTable.empty(0, L), S.GroupTable.empty(0, L), name)


# ---------------------------------------------------------------------------------------------------------------
# the tables

def edges_table():
    """Targets at the first visited node, the warp edges 31 / 32 / 63, the chunk edges 255 / 256 / 257, alone in a
    chunk of skipped nodes (600 in 512..767), and in the partial last warp just before the last visited node
    (N = 1350: nodes 1344..1349, last visited 1347)."""
    N, L = 1350, 6
    rng = np.random.default_rng(11)
    targets = [0, 31, 32, 63, 255, 256, 257, 600, 1346]
    peaks = [100, 900]
    kinds = sprinkle(N, rng, targets + peaks)
    kinds[512:768] = rng.choice(SKIP_KINDS, 256)
    kinds[600] = kinds[768] = FIT
    kinds[1347] = FIT
    kinds[1348:] = [NIL, UNSCHED]
    P = antichain(kinds, L, targets, peaks)
    nt = build_nodes(L, kinds, P, {})
    t = Table("edges", _snap(nt, "edges"), 1.0, targets)
    return _finish(t, [(x, scalar_mask(L), k % L) for k, x in enumerate(targets)])


def leading_skip_table(N=3200, L=5):
    """40 skipped nodes first; every visited prefix is negative on some lane.  Needs <= 0 on every lane are met by
    the targets (negative antichain values) or by nothing; a scan that tests a skipped position (its prefix is all
    zeros) would accept the need of -1 or 0 on every lane."""
    rng = np.random.default_rng(12)
    targets = [40, 1500, 2100, 3150]
    peaks = [700, 2600]
    kinds = sprinkle(N, rng, targets + peaks)
    kinds[:40] = rng.choice(SKIP_KINDS, 40)
    kinds[40] = FIT
    P = antichain(kinds, L, targets, peaks, hi={d: -30 - d for d in range(2, L)})
    fit = np.flatnonzero(kinds == FIT)
    pos = {i: k for k, i in enumerate(fit)}
    for k, t in enumerate(targets):       # shift the antichain below zero: cpu -60.., memory -40..
        P[pos[t]][0] -= 160
        P[pos[t]][1] -= 140 + 20 * len(targets)
    P[pos[peaks[0]]][2:] = [PEAK] * (L - 2)
    nt = build_nodes(L, kinds, P, {})
    t = Table("leading_skip", _snap(nt, "leading_skip"), 1.0, targets)
    _finish(t, [(x, scalar_mask(L), k % L) for k, x in enumerate(targets)])
    t.needs.append(([-1] * L, 0, "false", None))            # the all-zero prefix at a skipped node would meet it
    t.needs.append(([0] * L, scalar_mask(L), "false", None))
    return t


def scalar_table():
    """Scalar keys that some prefixes lack.  Lane 4's key arrives at node 400: a need on it that is not 0 cannot be
    met before (the decoy at 200 matches every other lane of the target at 500).  Lane 5's key arrives at node 300
    and every prefix that has it is negative, its maximum -1 at node 350: a need of 0 is met only where the key is
    still absent (target 150), a need of -1 nowhere."""
    N, L = 900, 6
    rng = np.random.default_rng(13)
    targets = [150, 500, 600]
    a1, decoy, q, a0 = 50, 200, 350, 450
    kinds = sprinkle(N, rng, targets + [a1, decoy, q, a0])
    key_from = {4: 400, 5: 300}
    fit = np.flatnonzero(kinds == FIT)
    P = antichain(kinds, L, targets, [a0, a1])
    pos = {i: k for k, i in enumerate(fit)}
    P[pos[decoy]] = list(P[pos[500]])
    P[pos[q]][5] = -1
    P[pos[a0]][4], P[pos[a0]][5] = PEAK, -3
    P[pos[500]][4], P[pos[500]][5] = -7, -5
    P[pos[600]][4], P[pos[600]][5] = -8, -2
    nt = build_nodes(L, kinds, P, key_from)
    t = Table("scalar_keys", _snap(nt, "scalar_keys"), 1.0, targets)
    _finish(t, [(150, 1 << 5, 0), (500, 1 << 4, 4), (600, 1 << 5, 5), (600, (1 << 4) | (1 << 5), 1)])
    need, npres, _, _ = t.needs[0]
    t.needs.append((need[:5] + [-1], npres, "false", None))      # the same need with -1 on the key target 150 lacks
    return t


def wrap_table():
    """Memory terms of +2^56 on every fit node: the running sum passes 2^63 at the 128th and wraps.  Target 110
    lies before the wrap; target 160 after it, with a memory need 1 above the wrapped prefix at node 150."""
    N, L = 220, 4
    kinds = np.full(N, FIT)
    kinds[[180, 190]] = [NIL, TAINTS_ERR]
    targets, a0 = [110, 160], 140
    fit = list(np.flatnonzero(kinds == FIT))
    pos = {i: k for k, i in enumerate(fit)}
    P = [[LOW - k] * L for k in range(len(fit))]
    P[pos[110]] = [100, 0, 60, 70]
    P[pos[160]] = [200, 0, 60, 70]
    P[pos[a0]] = [1000, 0, 600, 700]
    nt = build_nodes(L, kinds, P, {}, raw={1: [1 << 56] * len(fit)})
    t = Table("wrap", _snap(nt, "wrap"), 1.0, targets)
    pre, keys, _ = ref_prefixes(t, SEL, TOL, 1.0)
    assert pre[1, 126] > 0 > pre[1, 127]
    need = [100, 100 << 56, 60, 70]
    t.needs += [(need, 0, "true", 110), ([101] + need[1:], 0, "false", None)]
    need = [200, int(pre[1, 150]) + 1, 60, 70]
    t.needs += [(need, 0, "true", 160), ([200, int(pre[1, 160]) + 1, 60, 70], 0, "false", None)]
    return t


def real_alloc_table():
    """The antichain design at percent 0.7 with real allocatable values, so every term goes through
    int64(float32(alloc) * 0.7)."""
    N, L = 800, 5
    rng = np.random.default_rng(14)
    targets = [0, 31, 32, 300, 640]
    peaks = [150, 500]
    kinds = sprinkle(N, rng, targets + peaks)
    P = antichain(kinds, L, targets, peaks)
    alloc = [16777217, (1 << 40) | 1, 33554433, 110, 7]
    nt = build_nodes(L, kinds, P, {}, pct=0.7, alloc=alloc, seed=14)
    t = Table("real_alloc", _snap(nt, "real_alloc"), 0.7, targets)
    return _finish(t, [(x, scalar_mask(L), k % L) for k, x in enumerate(targets)])


def two_node_table():
    """N = 2: node 1 tops every lane, but only node 0's prefix lacks the scalar key, so a need of 0 on it is met
    there and not at the last prefix."""
    L = 5
    nt = S.NodeTable.empty(2, L)
    nt.label_mask[:] = 1
    nt.requested[:3, 0], nt.pod_count[0] = -5, -5
    nt.requested[:3, 1], nt.pod_count[1] = -3, -3
    nt.alloc_present[1] = nt.req_present[1] = 1 << 4
    nt.requested[4, 1] = 4               # term -4
    t = Table("two_nodes", _snap(nt, "two_nodes"), 1.0, [0])
    t.needs += [([5, 5, 5, 5, 0], 1 << 4, "true", 0), ([6, 5, 5, 5, 0], 1 << 4, "false", None)]
    return t


def one_node_table():
    L = 4
    nt = S.NodeTable.empty(1, L)
    nt.label_mask[:] = 1
    nt.requested[:3, 0], nt.pod_count[0] = -5, -5
    return Table("one_node", _snap(nt, "one_node"), 1.0, [])


def big_table(bump=False, N=3500, L=16):
    """16 lanes, 14 prefix chunks, 4 replay blocks of 1024.  Targets sit in the middle blocks, each block's maximum
    on every lane >= 2, and on cpu or memory, is exactly a target's need; the peaks are in blocks 0 and 3.
    bump=True adds 70 ephemeral-storage terms of about +2^56 and then 70 of about -2^56 in block 0: the running sum
    passes 2^62 there and comes back (the replay then runs without its block cache)."""
    rng = np.random.default_rng(15)
    targets = [1100, 1500, 2047, 2048, 2500, 2999]
    peaks = [500, 3300]
    kinds = sprinkle(N, rng, targets + peaks)
    if bump:
        kinds[100:250] = FIT
    P = antichain(kinds, L, targets, peaks)
    raw = None
    if bump:
        fit = list(np.flatnonzero(kinds == FIT))
        pos = {i: k for k, i in enumerate(fit)}
        terms = [P[k][2] - (P[k - 1][2] if k else 0) for k in range(len(fit))]
        for j in range(70):     # 2^56 - 2: with the design's own step of -1 a term stays within +-2^56
            terms[pos[100 + j]] += (1 << 56) - 2
            terms[pos[170 + j]] -= (1 << 56) - 2
        raw = {2: terms}
    nt = build_nodes(L, kinds, P, {}, raw=raw)
    t = Table("big_bump" if bump else "big", _snap(nt, "big_bump" if bump else "big"), 1.0, targets)
    return _finish(t, [(x, scalar_mask(L), [0, 1, 3, 7, 15, 1][k]) for k, x in enumerate(targets)])


@functools.lru_cache(maxsize=None)
def tables():
    """Every designed table; each has needs that only the full scan decides, both ways."""
    return [edges_table(), leading_skip_table(), scalar_table(), wrap_table(), real_alloc_table(), two_node_table(),
            big_table(), big_table(bump=True)]


_PRE = {}


def ref_prefixes(table, sel, tol, pct):
    key = (id(table.nodes), sel, tol, float(pct))
    if key not in _PRE:
        _PRE[key] = prefixes(table.nodes, sel, tol, pct)
    return _PRE[key]


def random_needs(table, sel, tol, pct, n, seed):
    """Needs around the reference prefixes: a prefix with small changes, the lane-wise max or min of two prefixes,
    random scalar key sets.  Returns need[L, n] int64 and npres[n] uint32."""
    rng = np.random.default_rng(seed)
    pre, keys, vis = ref_prefixes(table, sel, tol, pct)
    L = table.lanes
    idx = np.flatnonzero(vis)
    need = np.zeros((L, n), np.int64)
    npres = np.zeros(n, np.uint32)
    if len(idx) == 0:
        return need, npres
    for j in range(n):
        a, b = (int(x) for x in rng.choice(idx, 2))
        mode = j % 3
        if mode == 0:
            v = [int(pre[d, a]) + int(rng.choice([-1, 0, 0, 1])) for d in range(L)]
        elif mode == 1:
            v = [max(int(pre[d, a]), int(pre[d, b])) for d in range(L)]
        else:
            v = [min(int(pre[d, a]), int(pre[d, b])) + int(rng.choice([0, 1])) for d in range(L)]
        m = int(rng.integers(0, 1 << L)) & scalar_mask(L)
        for d in range(4, L):
            if rng.random() < 0.15:
                v[d] = 0
        need[:, j] = [i64(x) for x in v]
        npres[j] = m
    return need, npres


def need_arrays(needs, L):
    need = np.array([[i64(x) for x in n[0]] for n in needs], np.int64).reshape(-1, L).T.copy()
    npres = np.array([n[1] for n in needs], np.uint32)
    return need, npres


def reference_answers(table, sel, tol, pct, need, npres):
    pre, keys, vis = ref_prefixes(table, sel, tol, pct)
    return np.array([first_hit(pre, keys, vis, need[:, j], int(npres[j])) >= 0 for j in range(need.shape[1])])
