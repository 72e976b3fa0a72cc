/* preempt_host_ports_ref.c — TEST INFRASTRUCTURE: the CPU restatement of bs_preempt and bs_preempt_walk under the
 * PodFitsHostPorts filter (include/bsched.h bs_upload_bound_host_ports), linked against oracle/libbs_oracle.so.
 * tests/preempt_host_ports_ref.py compiles and binds it.
 *
 * It restates upstream's selectVictimsOnNode / podPassesFiltersOnNode with NodeInfo's HostPortInfo (k8s v1.17.5
 * [upstream, from memory]): each node's used ports are a SET of (ip, protocol, port) tuples.  Add inserts a tuple,
 * Remove deletes it whoever else holds it, and CheckConflict compares one wanted tuple with every used one (the same
 * protocol and port, and "0.0.0.0" on either side or the same ip).  The engine's conflict masks are not used: the
 * packed masks are only decoded into tuples through the dictionary.  Nominated pods are added to a clone of the node
 * at filter time (addNominatedPods), so an eviction never removes their tuples.
 *
 * Resources, RemovePod, the reprieve order and the pick are tests/preempt_pdb_ref.c's, and the walk's state handling is
 * tests/preempt_walk_ref.c's: both are included for their helpers.  With no ports anywhere the answers are theirs. */
#include "preempt_walk_ref.c"

#define BSHP_MAX 64
#define BSHP_IP_ANY 0u

typedef struct {
  uint32_t ip, protocol;
  int32_t port;
} hp_tuple;

/* HostPortInfo: a set of tuples */
typedef struct {
  uint32_t n;
  hp_tuple t[BSHP_MAX];
} hp_set;

typedef struct {
  uint32_t n_entries;
  const uint32_t* ip;
  const uint32_t* protocol;
  const int32_t* port;
} bshp_dict;

static int same_tuple(hp_tuple a, hp_tuple b) { return a.ip == b.ip && a.protocol == b.protocol && a.port == b.port; }

static void hpi_add(hp_set* s, hp_tuple x) {
  for (uint32_t i = 0; i < s->n; ++i)
    if (same_tuple(s->t[i], x)) return;
  s->t[s->n++] = x;
}

static void hpi_remove(hp_set* s, hp_tuple x) {
  for (uint32_t i = 0; i < s->n; ++i)
    if (same_tuple(s->t[i], x)) {
      s->t[i] = s->t[--s->n];
      return;
    }
}

/* HostPortInfo.CheckConflict for one wanted tuple */
static int hpi_conflict(const hp_set* s, hp_tuple x) {
  for (uint32_t i = 0; i < s->n; ++i) {
    const hp_tuple u = s->t[i];
    if (u.protocol != x.protocol || u.port != x.port) continue;
    if (x.ip == BSHP_IP_ANY || u.ip == BSHP_IP_ANY || u.ip == x.ip) return 1;
  }
  return 0;
}

/* the tuples of a packed mask */
static void decode(const bshp_dict* d, uint64_t mask, hp_set* out) {
  out->n = 0;
  for (uint32_t k = 0; k < d->n_entries; ++k)
    if ((mask >> k) & 1u) hpi_add(out, (hp_tuple){d->ip[k], d->protocol[k], d->port[k]});
}

static void add_all(hp_set* s, const hp_set* x) {
  for (uint32_t i = 0; i < x->n; ++i) hpi_add(s, x->t[i]);
}

static void remove_all(hp_set* s, const hp_set* x) {
  for (uint32_t i = 0; i < x->n; ++i) hpi_remove(s, x->t[i]);
}

/* PodFitsHostPorts of a pod wanting `want` on a clone of `used` with the nominated pods' tuples added */
static int ports_fit(const hp_set* used, const hp_set* nom, const hp_set* want) {
  hp_set clone = *used;
  add_all(&clone, nom);
  for (uint32_t i = 0; i < want->n; ++i)
    if (hpi_conflict(&clone, want->t[i])) return 0;
  return 1;
}

/* pickOneNodeForPreemption over candidates [0, nc) in node order (tests/preempt_pdb_ref.c's staged filters) */
static int32_t pick_one(const bsp_bound* b, uint32_t nc, const uint32_t* coff, const uint32_t* cvict,
                        const uint32_t* cviol) {
  for (uint32_t c2 = 0; c2 < nc; ++c2)
    if (coff[c2 + 1] == coff[c2]) return (int32_t)c2;
  if (!nc) return -1;
  uint32_t* set = malloc(nc * 4);
  uint32_t ns = 0, min_viol = UINT32_MAX;
  for (uint32_t c2 = 0; c2 < nc; ++c2) {
    if (cviol[c2] < min_viol) { min_viol = cviol[c2]; ns = 0; }
    if (cviol[c2] == min_viol) set[ns++] = c2;
  }
  if (ns > 1) {
    int32_t min_hp = INT32_MAX;
    uint32_t m = 0;
    for (uint32_t j = 0; j < ns; ++j) {
      const int32_t hp = b->priority[cvict[coff[set[j]]]];
      if (hp < min_hp) { min_hp = hp; m = 0; }
      if (hp == min_hp) set[m++] = set[j];
    }
    ns = m;
  }
  if (ns > 1) {
    int64_t min_sum = INT64_MAX;
    uint32_t m = 0;
    for (uint32_t j = 0; j < ns; ++j) {
      int64_t s = 0;
      for (uint32_t q = coff[set[j]]; q < coff[set[j] + 1]; ++q) s += (int64_t)b->priority[cvict[q]] + 2147483648LL;
      if (s < min_sum) { min_sum = s; m = 0; }
      if (s == min_sum) set[m++] = set[j];
    }
    ns = m;
  }
  if (ns > 1) {
    uint32_t min_n = UINT32_MAX, m = 0;
    for (uint32_t j = 0; j < ns; ++j) {
      const uint32_t cnt = coff[set[j] + 1] - coff[set[j]];
      if (cnt < min_n) { min_n = cnt; m = 0; }
      if (cnt == min_n) set[m++] = set[j];
    }
    ns = m;
  }
  uint32_t best = set[0];
  int64_t latest = INT64_MIN;
  for (uint32_t j = 0; j < ns; ++j) {
    int32_t hp = INT32_MIN;
    for (uint32_t q = coff[set[j]]; q < coff[set[j] + 1]; ++q)
      if (b->priority[cvict[q]] > hp) hp = b->priority[cvict[q]];
    int64_t earliest = INT64_MAX;
    for (uint32_t q = coff[set[j]]; q < coff[set[j] + 1]; ++q)
      if (b->priority[cvict[q]] == hp && b->start_ns[cvict[q]] < earliest) earliest = b->start_ns[cvict[q]];
    if (j == 0 || earliest > latest) { latest = earliest; best = set[j]; }
  }
  free(set);
  return (int32_t)best;
}

/* Preemption of pod p against nodes `nd`, bound rows `b` (row v holds the tuples of ports[v]), each node's bound set
 * used[i] and nominated set nom[i].  Writes the node (-1 none), the candidate count and the victims (row indices of b,
 * reprieve order) and returns the victim count. */
static uint32_t preempt_one(const bso_nodes* nd, const bso_pods* pd, const bsp_bound* b, const bshp_dict* d,
                            const uint64_t* ports, const hp_set* used, const hp_set* nom, const hp_set* want,
                            uint32_t p, int32_t* node_out, uint32_t* cand_out, uint32_t* victims) {
  const uint32_t N = nd->n, V = b->n;
  const int32_t prio = pd->priority[p];
  uint32_t* cnode = malloc((N + 1) * 4);
  uint32_t* coff = malloc((N + 2) * 4);
  uint32_t* cvict = malloc((V + 1) * 4);
  uint32_t* cviol = malloc((N + 1) * 4);
  uint32_t* pot = malloc((V + 1) * 4);
  uint32_t* tmp = malloc((V + 1) * 4);
  node_copy c;
  c.aff = malloc((nd->n_aff + 1) * 4);
  hp_set hp, row;
  uint32_t nc = 0;
  coff[0] = 0;
  for (uint32_t i = 0; i < N; ++i) {
    if (!node_might_help(nd, pd, p, i)) continue;   /* ErrPodNotFitsHostPorts is resolvable: not a reason to skip */
    uint32_t np = 0;
    int refused = 0;
    for (uint32_t v = 0; v < V; ++v) {
      if (b->node[v] != i || b->priority[v] >= prio) continue;
      if (remove_pod(pd->gid[p], b->gid[v], b->flags[v]) != BSR_ALLOW) refused = 1;
      pot[np++] = v;
    }
    if (refused) continue;
    copy_node(&c, nd, i);
    hp = used[i];
    for (uint32_t j = 0; j < np; ++j) {   /* removePod: Requests and HostPortInfo.Remove of every tuple */
      apply(&c, b, pot[j], -1);
      decode(d, ports[pot[j]], &row);
      remove_all(&hp, &row);
    }
    if (!bso_fit_eval(&c.nd, pd, p, 0, NULL) || !ports_fit(&hp, &nom[i], want)) continue;
    sort_more_important(b, pot, np);
    split_violating(b, pot, tmp, np);
    uint32_t nv = 0, nviol = 0;
    for (uint32_t j = 0; j < np; ++j) {   /* reprievePod: addPod, the filters, removePod when they fail */
      decode(d, ports[pot[j]], &row);
      apply(&c, b, pot[j], +1);
      add_all(&hp, &row);
      if (bso_fit_eval(&c.nd, pd, p, 0, NULL) && ports_fit(&hp, &nom[i], want)) continue;
      apply(&c, b, pot[j], -1);
      remove_all(&hp, &row);
      cvict[coff[nc] + nv++] = pot[j];
      if (b->flags[pot[j]] & BSR_PDB_VIOLATING) ++nviol;
    }
    cviol[nc] = nviol;
    cnode[nc] = i;
    coff[nc + 1] = coff[nc] + nv;
    ++nc;
  }
  *cand_out = nc;
  const int32_t pick = pick_one(b, nc, coff, cvict, cviol);
  uint32_t nv = 0;
  if (pick < 0) {
    *node_out = -1;
  } else {
    *node_out = (int32_t)cnode[pick];
    nv = coff[pick + 1] - coff[pick];
    memcpy(victims, cvict + coff[pick], (size_t)nv * 4);
  }
  free(c.aff); free(tmp); free(pot); free(cviol); free(cvict); free(coff); free(cnode);
  return nv;
}

/* bs_preempt under the filter: used[N] the node side's masks, ports[V] the bound side's, want[P] the pod side's.
 * victims[k * vstride ..] as tests/preempt_pdb_ref.c's bsp_preempt. */
void bshp_preempt(const bso_nodes* nd, const bso_pods* pd, const bsp_bound* b, const bshp_dict* d,
                  const uint64_t* used, const uint64_t* ports, const uint64_t* want, const uint32_t* pods, uint32_t n,
                  int32_t* node_out, uint32_t* nv_out, uint32_t* cand_out, uint32_t* victims, uint32_t vstride) {
  const uint32_t N = nd->n;
  hp_set* sets = malloc(((size_t)N + 1) * sizeof(hp_set));
  hp_set* nom = calloc((size_t)N + 1, sizeof(hp_set));
  for (uint32_t i = 0; i < N; ++i) decode(d, used[i], &sets[i]);
  uint32_t* vict = malloc(((size_t)b->n + 1) * 4);
  hp_set w;
  for (uint32_t k = 0; k < n; ++k) {
    decode(d, want[pods[k]], &w);
    nv_out[k] = preempt_one(nd, pd, b, d, ports, sets, nom, &w, pods[k], &node_out[k], &cand_out[k], vict);
    for (uint32_t q = 0; q < nv_out[k] && q < vstride; ++q) victims[(size_t)k * vstride + q] = vict[q];
  }
  free(vict); free(nom); free(sets);
}

/* bs_preempt_walk under the filter, as tests/preempt_walk_ref.c's bsw_walk: per node a bound set (evictions remove the
 * victims' tuples) and a nominated set (nominations add the preemptor's), both saved and restored with a gang unit. */
uint32_t bshp_walk(const bso_nodes* nd0, const bso_pods* pd, const bsp_bound* b, const bshp_dict* d,
                   const uint64_t* used, const uint64_t* ports, const uint64_t* want, const uint32_t* pods, uint32_t n,
                   const uint8_t* unit_last, int gang, int32_t* node_out, uint32_t* nv_out, uint32_t* cand_out,
                   uint32_t* outcome, uint32_t* victims, int32_t* evicted_by) {
  const uint32_t N = nd0->n, L = nd0->lanes, V = b->n;
  const size_t nl = (size_t)L * N + 1;
  int64_t* req = malloc(nl * 8);
  int64_t* req_save = malloc(nl * 8);
  int32_t* pc = malloc(((size_t)N + 1) * 4);
  int32_t* pc_save = malloc(((size_t)N + 1) * 4);
  uint32_t* rp = malloc(((size_t)N + 1) * 4);
  uint32_t* rp_save = malloc(((size_t)N + 1) * 4);
  int32_t* ev_save = malloc(((size_t)V + 1) * 4);
  const size_t sb = ((size_t)N + 1) * sizeof(hp_set);
  hp_set* bset = malloc(sb);
  hp_set* nset = calloc((size_t)N + 1, sizeof(hp_set));
  hp_set* bset_save = malloc(sb);
  hp_set* nset_save = malloc(sb);
  memcpy(req, nd0->requested, (size_t)L * N * 8);
  memcpy(pc, nd0->pod_count, (size_t)N * 4);
  memcpy(rp, nd0->req_present, (size_t)N * 4);
  for (uint32_t i = 0; i < N; ++i) decode(d, used[i], &bset[i]);
  bso_nodes nd = *nd0;
  nd.requested = req;
  nd.pod_count = pc;
  nd.req_present = rp;
  const size_t vl = (size_t)L * V + 1;
  uint32_t* l_node = malloc(((size_t)V + 1) * 4);
  int64_t* l_req = malloc(vl * 8);
  uint32_t* l_rp = malloc(((size_t)V + 1) * 4);
  int32_t* l_gid = malloc(((size_t)V + 1) * 4);
  int32_t* l_prio = malloc(((size_t)V + 1) * 4);
  int64_t* l_start = malloc(((size_t)V + 1) * 8);
  uint8_t* l_flags = malloc((size_t)V + 1);
  uint64_t* l_ports = malloc(((size_t)V + 1) * 8);
  uint32_t* l_orig = malloc(((size_t)V + 1) * 4);
  uint32_t* vict = malloc(((size_t)V + 1) * 4);
  node_copy c;
  c.aff = malloc((nd.n_aff + 1) * 4);
  hp_set w, row;
  for (uint32_t v = 0; v < V; ++v) evicted_by[v] = -1;
  uint32_t voff = 0, voff_save = 0, unit_first = 0;
  int failed = 0;
  for (uint32_t i = 0; i < n; ++i) {
    if (i == unit_first && gang) {
      memcpy(req_save, req, (size_t)L * N * 8);
      memcpy(pc_save, pc, (size_t)N * 4);
      memcpy(rp_save, rp, (size_t)N * 4);
      memcpy(ev_save, evicted_by, (size_t)V * 4);
      memcpy(bset_save, bset, (size_t)N * sizeof(hp_set));
      memcpy(nset_save, nset, (size_t)N * sizeof(hp_set));
      voff_save = voff;
    }
    uint32_t m = 0;
    for (uint32_t v = 0; v < V; ++v) {
      if (evicted_by[v] >= 0) continue;
      l_node[m] = b->node[v];
      l_rp[m] = b->req_present[v];
      l_gid[m] = b->gid[v];
      l_prio[m] = b->priority[v];
      l_start[m] = b->start_ns[v];
      l_flags[m] = b->flags[v];
      l_ports[m] = ports[v];
      l_orig[m] = v;
      ++m;
    }
    for (uint32_t dd = 0; dd < L; ++dd)
      for (uint32_t k = 0; k < m; ++k) l_req[(size_t)dd * m + k] = b->req[(size_t)dd * V + l_orig[k]];
    const bsp_bound live = {m, L, l_node, l_req, l_rp, l_gid, l_prio, l_start, l_flags};
    const uint32_t p = pods[i];
    decode(d, want[p], &w);
    int32_t node;
    uint32_t cand;
    const uint32_t nv = preempt_one(&nd, pd, &live, d, l_ports, bset, nset, &w, p, &node, &cand, vict);
    cand_out[i] = cand;
    if (node < 0) {
      node_out[i] = -1;
      nv_out[i] = 0;
      outcome[i] = BSW_NONE;
      failed = 1;
    } else {
      node_out[i] = node;
      nv_out[i] = nv;
      outcome[i] = BSW_NOMINATED;
      copy_node(&c, &nd, (uint32_t)node);
      for (uint32_t j = 0; j < nv; ++j) {   /* NodeInfo.RemovePod: Requests and the tuples */
        const uint32_t v = l_orig[vict[j]];
        victims[voff++] = v;
        evicted_by[v] = (int32_t)i;
        apply(&c, b, v, -1);
        decode(d, ports[v], &row);
        remove_all(&bset[node], &row);
      }
      for (uint32_t dd = 0; dd < L; ++dd) req[(size_t)dd * N + node] = c.requested[dd];
      pc[node] = c.pod_count;
      for (uint32_t dd = 0; dd < L; ++dd) {   /* nominate: the oracle's assume, and the pod's tuples */
        if (dd == 3) continue;
        if (dd >= 4 && !(pd->req_present[p] & (1u << dd))) continue;
        req[(size_t)dd * N + node] += pd->req[(size_t)dd * pd->n + p];
        if (dd >= 4) rp[node] |= 1u << dd;
      }
      pc[node] += 1;
      add_all(&nset[node], &w);
    }
    if (!unit_last[i]) continue;
    if (gang && failed) {
      memcpy(req, req_save, (size_t)L * N * 8);
      memcpy(pc, pc_save, (size_t)N * 4);
      memcpy(rp, rp_save, (size_t)N * 4);
      memcpy(evicted_by, ev_save, (size_t)V * 4);
      memcpy(bset, bset_save, (size_t)N * sizeof(hp_set));
      memcpy(nset, nset_save, (size_t)N * sizeof(hp_set));
      voff = voff_save;
      for (uint32_t k = unit_first; k <= i; ++k) {
        node_out[k] = -1;
        nv_out[k] = 0;
        outcome[k] = BSW_ROLLED_BACK;
      }
    }
    failed = 0;
    unit_first = i + 1;
  }
  free(c.aff); free(vict); free(l_orig); free(l_ports); free(l_flags); free(l_start); free(l_prio); free(l_gid);
  free(l_rp); free(l_req); free(l_node); free(nset_save); free(bset_save); free(nset); free(bset); free(ev_save);
  free(rp_save); free(rp); free(pc_save); free(pc); free(req_save); free(req);
  return voff;
}
