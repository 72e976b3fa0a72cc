/* preempt_ref.c — TEST INFRASTRUCTURE: the CPU restatement of bs_remove_pod and bs_preempt (include/bsched.h), built on
 * the oracle's fit predicate (oracle/bs_oracle.h: bso_fit_eval) and linked against oracle/libbs_oracle.so.
 * tests/native.py compiles it with the other restatements and tests/preempt_ref.py binds it.
 *
 * Preemption is restated the way upstream does it (k8s v1.17.5 genericScheduler.Preempt -> selectVictimsOnNode ->
 * pickOneNodeForPreemption, [upstream, from memory]): on a MUTATED one-node copy of each node, removing and re-adding
 * pods and calling the fit predicate after every step, then the pick's staged filters over the candidates in node
 * order.  The engine uses suffix sums instead; the two must agree. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "bs_oracle.h"

enum { BSR_ALLOW = 0, BSR_OFFLINE_ONLINE = 1, BSR_NOT_FOUND = 2, BSR_LOCKED = 3, BSR_SAME_GROUP = 4 };
#define BSR_LOCKED_FLAG 0x01u

typedef struct {
  uint32_t n, lanes;
  const uint32_t* node;
  const int64_t* req; /* [lanes][n] */
  const uint32_t* req_present;
  const int32_t* gid;
  const int32_t* priority;
  const int64_t* start_ns;
  const uint8_t* flags;
} bsr_bound;

/* core.PreemptRemovePod (core.go:203-260), gid_p / gid_v: group index, BSO_GID_NONE (no label) or BSO_GID_MISSING */
int bsr_remove_pod(int32_t gid_p, int32_t gid_v, uint8_t flags_v) {
  const int offline_remove = gid_v != BSO_GID_NONE;      /* :204 VerifyPodLabelSatisfied */
  const int offline_schedule = gid_p != BSO_GID_NONE;    /* :205 */
  if (!offline_schedule && !offline_remove) return BSR_ALLOW;        /* :213-215 */
  if (offline_schedule && !offline_remove) return BSR_OFFLINE_ONLINE; /* :216-218 */
  /* checkPreemption :220-240: fullNameToRemove, or "" with an error */
  int err = BSR_ALLOW;
  int32_t full_name_to_remove = -1;   /* "" */
  if (gid_v == BSO_GID_MISSING) err = BSR_NOT_FOUND;                 /* :222-225 */
  else if (flags_v & BSR_LOCKED_FLAG) err = BSR_LOCKED;              /* :234-238 */
  else full_name_to_remove = gid_v;
  if (!offline_schedule && offline_remove) return err;               /* :245-247 */
  /* :250-253: fullNameToSchedule names p's group; a missing group of p has no index and never equals a found one */
  if (gid_p >= 0 && full_name_to_remove == gid_p) return BSR_SAME_GROUP;
  return err;                                                        /* :254-256 */
}

/* The candidate filter standing in for nodesWherePreemptionMightHelp: the guards (core.go:606-617, :639), checkFit
 * (:741-759) and the absent-key rule (:688-690) — what no removal can change. */
static int node_might_help(const bso_nodes* nd, const bso_pods* pd, uint32_t p, uint32_t i) {
  if (nd->flags[i] & (BSO_NODE_NIL | BSO_NODE_NO_NODE | BSO_NODE_UNSCHEDULABLE | BSO_NODE_TAINTS_ERR)) return 0;
  const uint32_t aff = pd->aff_class ? pd->aff_class[p] : BSO_AFF_NONE;
  if (!bso_check_fit(nd, i, pd->sel_mask[p], pd->tol_mask[p], aff)) return 0;
  const uint32_t left_keys = nd->alloc_present[i] & nd->req_present[i];
  for (uint32_t d = 4; d < nd->lanes; ++d)
    if (((pd->req_present[p] >> d) & 1u) && pd->req[(size_t)d * pd->n + p] != 0 && !((left_keys >> d) & 1u)) return 0;
  return 1;
}

/* one mutable node: NodeInfo after Clone() */
typedef struct {
  bso_nodes nd;
  int64_t alloc[BSO_MAX_LANES], requested[BSO_MAX_LANES];
  int32_t pod_count;
  uint32_t alloc_present, req_present;
  uint64_t label, taint;
  uint8_t flags;
  uint32_t* aff;   /* [n_aff] */
} node_copy;

static void copy_node(node_copy* c, const bso_nodes* src, uint32_t i) {
  const uint32_t L = src->lanes, W = (src->n + 31) / 32;
  for (uint32_t d = 0; d < L; ++d) {
    c->alloc[d] = src->alloc[(size_t)d * src->n + i];
    c->requested[d] = src->requested[(size_t)d * src->n + i];
  }
  c->pod_count = src->pod_count[i];
  c->alloc_present = src->alloc_present[i];
  c->req_present = src->req_present[i];
  c->label = src->label_mask[i];
  c->taint = src->taint_mask[i];
  c->flags = src->flags[i];
  for (uint32_t a = 0; a < src->n_aff; ++a) c->aff[a] = (src->aff_bits[(size_t)a * W + (i >> 5)] >> (i & 31)) & 1u;
  c->nd.n = 1;
  c->nd.lanes = L;
  c->nd.alloc = c->alloc;
  c->nd.requested = c->requested;
  c->nd.pod_count = &c->pod_count;
  c->nd.alloc_present = &c->alloc_present;
  c->nd.req_present = &c->req_present;
  c->nd.label_mask = &c->label;
  c->nd.taint_mask = &c->taint;
  c->nd.flags = &c->flags;
  c->nd.n_aff = src->n_aff;
  c->nd.aff_bits = src->n_aff ? c->aff : NULL;
}

/* NodeInfo.RemovePod / AddPod on the copy: the pod's Requests on lanes 0-2 and its scalar keys, one pod fewer / more
 * (lane 3 of requested is not a pod's request) */
static void apply(node_copy* c, const bsr_bound* b, uint32_t v, int sign) {
  for (uint32_t d = 0; d < b->lanes; ++d) {
    if (d == 3) continue;
    if (d >= 4 && !((b->req_present[v] >> d) & 1u)) continue;
    c->requested[d] += sign * b->req[(size_t)d * b->n + v];
  }
  c->pod_count += sign;
}

/* MoreImportantPod: priority descending, then start time ascending; the bound-table index decides the rest */
static int more_important(const bsr_bound* b, uint32_t a, uint32_t c) {
  if (b->priority[a] != b->priority[c]) return b->priority[a] > b->priority[c];
  if (b->start_ns[a] != b->start_ns[c]) return b->start_ns[a] < b->start_ns[c];
  return a < c;
}

/* sort.Slice(potential, MoreImportantPod): an insertion sort (a node holds few pods) */
static void sort_more_important(const bsr_bound* b, uint32_t* a, uint32_t n) {
  for (uint32_t i = 1; i < n; ++i) {
    const uint32_t x = a[i];
    uint32_t j = i;
    while (j > 0 && more_important(b, x, a[j - 1])) { a[j] = a[j - 1]; --j; }
    a[j] = x;
  }
}

/* Preemption for pods[0..n): node_out[i] (-1 none), nv_out[i], cand_out[i] and victims[i * vstride ..] in reprieve
 * order.  OpenMP over preemptors (threads <= 0: all), each an independent what-if with buffers of its own. */
void bsr_preempt(const bso_nodes* nd, const bso_pods* pd, const bsr_bound* b, const uint32_t* pods, uint32_t n,
                 int32_t* node_out, uint32_t* nv_out, uint32_t* cand_out, uint32_t* victims, uint32_t vstride,
                 int threads) {
  const uint32_t N = nd->n, V = b->n;
  /* NodeInfo.Pods() per node, table order */
  uint32_t* row = calloc(N + 1, 4);
  uint32_t* list = malloc((V + 1) * 4);
  for (uint32_t v = 0; v < V; ++v) row[b->node[v] + 1]++;
  for (uint32_t i = 0; i < N; ++i) row[i + 1] += row[i];
  uint32_t* fill = malloc((N + 1) * 4);
  memcpy(fill, row, (N + 1) * 4);
  for (uint32_t v = 0; v < V; ++v) list[fill[b->node[v]]++] = v;
  if (threads <= 0) threads = bso_max_threads();
#pragma omp parallel num_threads(threads)
  {
  /* per candidate: its victims */
  uint32_t* cnode = malloc((N + 1) * 4);
  uint32_t* coff = malloc((N + 2) * 4);
  uint32_t* cvict = malloc((V + 1) * 4);
  uint32_t* pot = malloc((V + 1) * 4);
  node_copy c;
  c.aff = malloc((nd->n_aff + 1) * 4);
#pragma omp for schedule(dynamic, 4)
  for (uint32_t k = 0; k < n; ++k) {
    const uint32_t p = pods[k];
    const int32_t prio = pd->priority[p];
    uint32_t nc = 0;
    coff[0] = 0;
    for (uint32_t i = 0; i < N; ++i) {
      if (!node_might_help(nd, pd, p, i)) continue;
      /* potential victims: lower priority; every one must pass RemovePod */
      uint32_t np = 0;
      int refused = 0;
      for (uint32_t j = row[i]; j < row[i + 1]; ++j) {
        const uint32_t v = list[j];
        if (b->priority[v] >= prio) continue;
        if (bsr_remove_pod(pd->gid[p], b->gid[v], b->flags[v]) != BSR_ALLOW) refused = 1;
        pot[np++] = v;
      }
      if (refused) continue;
      copy_node(&c, nd, i);
      for (uint32_t j = 0; j < np; ++j) apply(&c, b, pot[j], -1);
      if (!bso_fit_eval(&c.nd, pd, p, 0, NULL)) continue;
      sort_more_important(b, pot, np);
      uint32_t nv = 0;
      for (uint32_t j = 0; j < np; ++j) {   /* reprievePod */
        apply(&c, b, pot[j], +1);
        if (bso_fit_eval(&c.nd, pd, p, 0, NULL)) continue;
        apply(&c, b, pot[j], -1);
        cvict[coff[nc] + nv++] = pot[j];
      }
      cnode[nc] = i;
      coff[nc + 1] = coff[nc] + nv;
      ++nc;
    }
    cand_out[k] = nc;
    /* pickOneNodeForPreemption over the candidates in node order */
    int32_t pick = -1;
    for (uint32_t c2 = 0; c2 < nc && pick < 0; ++c2)
      if (coff[c2 + 1] == coff[c2]) pick = (int32_t)c2;   /* a node without victims: returned at once */
    if (pick < 0 && nc) {
      uint32_t* set = malloc(nc * 4);
      uint32_t ns = 0;
      int32_t min_hp = INT32_MAX;   /* highest victim priority: the first victim's */
      for (uint32_t c2 = 0; c2 < nc; ++c2) {
        const int32_t hp = b->priority[cvict[coff[c2]]];
        if (hp < min_hp) { min_hp = hp; ns = 0; }
        if (hp == min_hp) set[ns++] = c2;
      }
      if (ns > 1) {   /* sum of priorities, each + MaxInt32 + 1 */
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
      if (ns > 1) {   /* fewest victims */
        uint32_t min_n = UINT32_MAX, m = 0;
        for (uint32_t j = 0; j < ns; ++j) {
          const uint32_t cnt = coff[set[j] + 1] - coff[set[j]];
          if (cnt < min_n) { min_n = cnt; m = 0; }
          if (cnt == min_n) set[m++] = set[j];
        }
        ns = m;
      }
      /* latest "earliest start time of the highest-priority victims"; the first one in order stays on ties */
      uint32_t best = set[0];
      int64_t latest = INT64_MIN;
      for (uint32_t j = 0; j < ns; ++j) {
        const int32_t hp = b->priority[cvict[coff[set[j]]]];
        int64_t earliest = INT64_MAX;
        for (uint32_t q = coff[set[j]]; q < coff[set[j] + 1]; ++q)
          if (b->priority[cvict[q]] == hp && b->start_ns[cvict[q]] < earliest) earliest = b->start_ns[cvict[q]];
        if (j == 0 || earliest > latest) { latest = earliest; best = set[j]; }
      }
      pick = (int32_t)best;
      free(set);
    }
    if (pick < 0) {
      node_out[k] = -1;
      nv_out[k] = 0;
      continue;
    }
    node_out[k] = (int32_t)cnode[pick];
    nv_out[k] = coff[pick + 1] - coff[pick];
    for (uint32_t q = 0; q < nv_out[k] && q < vstride; ++q) victims[(size_t)k * vstride + q] = cvict[coff[pick] + q];
  }
  free(c.aff); free(pot); free(cvict); free(coff); free(cnode);
  }
  free(fill); free(list); free(row);
}
