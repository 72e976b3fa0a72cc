"""TEST INFRASTRUCTURE — the designed cases of the group-sharded round, and one rank's shard of a whole state.

Snapshot.shard_groups cuts the three tables: the node and group tables are replicated, the pods of the rank's group
range (and the ungrouped pods with index % world == rank) stay, in table order, at local.meta["pod_index"].  shard()
cuts the side columns the same way: every pod half (the non-zero [2][P] column, the preference, locality, spread and
inter-pod pod classes, the MatchInterPodAffinity filter's pod classes, the PodFitsHostPorts filter's want masks) is
sliced by pod, every node half and every class table is replicated as it is.  A case is an engine_model.Model holding
the whole state with every side column, all six priority weights and both filters on, so that Model.expect gives every
output of a round on the whole snapshot and on a shard alike.

The cases (each one's rounds move admits and max_group through identical group row updates, group_updates):
  unbalanced    three groups hold three quarters of the pods;
  ungrouped     close to half of the pods have gid < 0 (GID_NONE and GID_MISSING) and follow index % world;
  empty_shard   only two of six groups hold pods and no pod is ungrouped: with three or four ranks a rank gets no pod
                and no group;
  many_groups   8200 groups (words_per_rank 257 > 256: every block of peer_push_kernel loops twice), every third
                group with pods;
  many_groups3  16400 groups (513 words: three trips);
  tail          77 groups, a bitmap tail of 13 bits;
  idle          100 groups of which only 42 hold pods, the others before, between and after them: no rank holds a
                pod of those, so every rank decides them with group_idle_admit_kernel and must agree with the oracle.
"""
from __future__ import annotations

import numpy as np

import engine_model as em
import host_ports_ref as hr
from randsnap import S, random_snapshot

L = 6
EVERY_OUTPUT = dict(score=True, fit_bitmap=True, filter=True, reasons=True, topk=8, priority_k=8)
ROUNDS = 3          # the loaded state, then two group row updates
CASES = ("unbalanced", "ungrouped", "empty_shard", "many_groups", "many_groups3", "tail", "idle")
WORLDS = (2, 3, 4)
PER_POD = ("prefilter", "feasible_count", "best_node", "best_score", "fit_rows", "score_rows", "filter_rows",
           "filter_code", "reason_rows", "interpod_rows", "host_port_rows", "topk_nodes", "topk_scores", "priority_nodes",
           "priority_scores")


def _gids(name, rng):
    """(P, N, G, gid [P]) of a case."""
    if name == "unbalanced":
        P, N, G = 1200, 256, 48
        gid = np.where(rng.random(P) < 0.75, rng.choice([5, 6, 30], P), rng.integers(0, G, P))
        gid = np.where(rng.random(P) < 0.08, S.GID_NONE, np.where(rng.random(P) < 0.02, S.GID_MISSING, gid))
    elif name == "ungrouped":
        P, N, G = 900, 200, 24
        gid = np.where(rng.random(P) < 0.35, S.GID_NONE,
                       np.where(rng.random(P) < 0.15, S.GID_MISSING, rng.integers(0, G, P)))
    elif name == "empty_shard":
        P, N, G = 300, 160, 6
        gid = np.where(rng.random(P) < 0.6, 1, 4)
    elif name == "many_groups":
        P, N, G = 2400, 128, 8200
        gid = np.where(rng.random(P) < 0.05, S.GID_NONE, 3 * rng.integers(0, G // 3, P))
    elif name == "many_groups3":
        P, N, G = 3000, 96, 16400
        gid = np.where(rng.random(P) < 0.05, S.GID_NONE, rng.integers(0, G, P))
    elif name == "tail":
        P, N, G = 700, 300, 77
        gid = np.where(rng.random(P) < 0.1, S.GID_NONE, rng.integers(0, G, P))
    elif name == "idle":
        P, N, G = 800, 200, 100
        held = np.r_[10:41, 60:71]
        gid = np.where(rng.random(P) < 0.1, S.GID_NONE, rng.choice(held, P))
    else:
        raise ValueError(name)
    return P, N, G, np.asarray(gid, np.int32)


def case(name, seed=None) -> em.Model:
    """The whole state of case `name`: its tables (groups resolved), every side column, all six priority weights and
    both filters on."""
    seed = CASES.index(name) + 11 if seed is None else seed
    rng = np.random.default_rng(seed)
    P, N, G, gid = _gids(name, rng)
    snap = random_snapshot(seed, P=P, N=N, G=G, L=L, aff=em.AFF)
    snap.pods.gid = gid
    snap = snap.resolve_groups()
    m = em.Model(L)
    m.nodes, m.pods, m.groups, m.aff = snap.nodes, snap.pods, snap.groups, snap.aff_bits
    k = int(rng.integers(0, 1 << 30))
    m.side["nz_node"], m.side["nz_pod"] = S.nonzero_requests(snap, k)
    c = S.node_preferences(snap, k + 1)
    m.side["pref_node"], m.side["pref_pod"] = (c[0], c[1]), (c[2], c[3])
    m.side["loc_node"], m.side["loc_pod"] = S.node_locality(snap, k + 2)
    m.side["spread_node"], m.side["spread_pod"] = S.node_spread(snap, k + 3)
    m.side["ipa_node"], m.side["ipa_pod"] = S.node_interpod(snap, k + 4)
    # with thousands of gangs, few carry terms: the restatement loops over every bound pod for each (pod, node)
    few = dict(one_per_host=0.01, ps_affine=0.01, self_affine=0.01) if G > 1000 else {}
    m.ipf_node, m.ipf_pod = S.node_interpod_filter(snap, k + 5, **few)
    m.weights = (1, 0, 1)
    m.ratio = (em.RATIO_ON[0], em.RATIO_ON[1], [1, 1, 0, 0] + [1] * (L - 4), em.RATIO_ON[3])
    m.pw, m.lw, m.w_spread, m.w_ipa = em.PW, em.LW, em.W_SPREAD, em.W_IPA
    m.ipf_on = m.ipf_round = True
    m.hp_node, m.hp_pod = hr.random_columns(snap, k + 6)
    m.hp_on = m.hp_round = True
    return m


def _pod_half(name, cols, idx):
    if name == "nz":
        return np.ascontiguousarray(cols[:, idx])
    if name == "pref":
        return cols[0][idx], cols[1][idx]
    if name == "loc":
        return cols[0][idx], cols[1], cols[2], cols[3][idx]
    if name == "spread":
        return cols[idx]
    return cols[0][idx], cols[1]     # ipa and the filter: (pod classes, class table)


def shard(m: em.Model, rank: int, world: int):
    """(rank's Model, pod_index, (g0, g1)): the shard's pod table and pod halves, everything else as in m."""
    local = m.snapshot().shard_groups(rank, world)
    idx = local.meta["pod_index"]
    s = em.Model(m.lanes)
    s.__dict__.update({k: v for k, v in m.__dict__.items() if k not in ("side", "pods", "ipf_pod", "hp_pod")})
    s.pods = local.pods
    s.side = {k: (v if k.endswith("_node") else _pod_half(k.split("_")[0], v, idx)) for k, v in m.side.items()}
    s.ipf_pod = _pod_half("ipf", m.ipf_pod, idx)
    s.hp_pod = np.ascontiguousarray(m.hp_pod[idx])
    return s, idx, local.meta["group_range"]


def group_updates(m: em.Model):
    """ROUNDS - 1 group row updates (idx, rows), the same on every rank.  Each takes up to 12 groups with a pod that
    fits and flips them (admitted: min_member 1000 and nothing matched or scheduled; else fully matched), and knocks
    the round's max_group down to nothing matched or scheduled, so that admits and max_group move."""
    rng = np.random.default_rng(m.groups.n)
    G = m.groups.n
    gid = m.pods.gid
    ok = (gid >= 0) & (gid < G)
    out, groups = [], m.groups
    for _ in range(ROUNDS - 1):
        r = with_groups(m, groups).expect({})
        fits = np.bincount(gid[ok], weights=((r["prefilter"] == 0) & (r["feasible_count"] > 0))[ok], minlength=G) > 0
        cand = np.flatnonzero(fits)
        pick = rng.choice(cand, min(12, len(cand)), replace=False) if len(cand) else []
        top = r["max_group"]
        idx = np.unique(np.r_[pick, [top] if top >= 0 else []]).astype(np.uint32)
        rows = groups.take(idx).copy()
        admitted = r["admit"][idx] == S.ADMIT
        rows.min_member = np.where(admitted, 1000, rows.min_member).astype(np.uint32)
        rows.matched = np.where(admitted, 0, rows.min_member).astype(np.uint32)
        rows.scheduled[:] = 0
        if top >= 0:
            rows.matched[int(np.searchsorted(idx, top))] = 0
        out.append((idx, rows))
        groups = em._apply_rows(groups, idx, rows)
    return out


def with_groups(m: em.Model, groups) -> em.Model:
    """A copy of m with another group table."""
    c = em.Model(m.lanes)
    c.__dict__.update(m.__dict__)
    c.groups = groups
    return c


def updated(m: em.Model, upd) -> em.Model:
    """A copy of m after the group row update upd = (idx, rows)."""
    return with_groups(m, em._apply_rows(m.groups, *upd))


def idle_groups(m: em.Model) -> np.ndarray:
    """[G] bool: groups no pod of the whole table names."""
    gid = m.pods.gid
    return np.bincount(gid[(gid >= 0) & (gid < m.groups.n)], minlength=m.groups.n) == 0


def first_diff(full: dict, got: dict, idx, g0: int, g1: int, idle) -> str | None:
    """The first output of a shard's round `got` (keyed as Model.expect keys them, any subset of the per-pod rows)
    that differs from the whole snapshot's round `full` restricted to the shard: the per-pod rows at pod_index,
    admit and new_denied on the rank's own group range and on the groups no rank holds pods of, max_group and
    max_finished as they are, order as the whole order filtered to the shard, rank as its dense re-ranking."""
    for k in PER_POD:
        if k in got and not np.array_equal(np.asarray(got[k]), np.asarray(full[k])[idx]):
            g, w = np.asarray(got[k]), np.asarray(full[k])[idx]
            if g.shape != w.shape:
                return f"{k}: shape {g.shape} != {w.shape}"
            return f"{k}: first differing rows {np.unique(np.argwhere(g != w)[:, 0])[:4].tolist()}"
    for k in ("admit", "new_denied"):
        g, w = np.asarray(got[k]), np.asarray(full[k])
        for what, sel in (("own range", slice(g0, g1)), ("groups without pods", idle)):
            if not np.array_equal(g[sel], w[sel]):
                at = np.flatnonzero(g[sel] != w[sel])[:4]
                return f"{k} on {what}: first differing positions {at.tolist()}"
    for k in ("max_group", "max_finished"):
        if int(got[k]) != int(full[k]):
            return f"{k}: {int(got[k])} != {int(full[k])}"
    order = np.asarray(full["order"])
    want = order[np.isin(order, idx)]
    if not np.array_equal(idx[np.asarray(got["order"], np.int64)], want):
        return "order: not the whole order filtered to the shard"
    if not np.array_equal(np.asarray(got["rank"]), np.unique(np.asarray(full["rank"])[idx], return_inverse=True)[1]):
        return "rank: not the dense re-ranking of the whole rank"
    return None


def admit_bits(words: np.ndarray, G: int) -> np.ndarray:
    """[G] bool from one rank's bitmap words."""
    return np.unpackbits(np.ascontiguousarray(words, np.uint32).view(np.uint8), bitorder="little")[:G].astype(bool)
