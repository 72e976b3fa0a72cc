/* interpod_walk_ref.c — TEST INFRASTRUCTURE: the MatchInterPodAffinity filter in the walks (include/bsched.h
 * bs_upload_pod_interpod_placed), restated on the packed columns of the filter's two sides and the placed side.  No
 * presence tables: for each (pod, node) it loops over the bound pods and the pods the walk has assumed so far, the
 * latter with their placed classes, in the order of the four steps.  bsr_ipw_choose / bsr_ipw_assumed are a chooser /
 * assume hook pair for tests/replay_priority_ref.c's bsr_replay_choose: they wrap another pair (first fit, priority,
 * ratio, locality, or tests/host_ports_ref.c's pair around one of those) and keep the list of assumed pods.
 * tests/interpod_walk_ref.py compiles it into a library of its own. */
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>

#include "bs_oracle.h"
#include "bs_ref.h"

#define BSR_IPW_NONE 0xffffffffu
#define BSR_IPW_TOPO_NONE 0xffffffffu
enum { BSR_IPW_AFFINITY = 0, BSR_IPW_ANTI = 1, BSR_IPW_EXISTING = 2 };

/* A class table: class c's entries are [off[c], off[c + 1]) of term / own / match (own NULL: a filter class, whose
 * entries are (term, role) in term / role). */
typedef struct {
  const uint32_t* off;
  const uint32_t* term;
  const int32_t* own;
  const uint8_t* match;
} bsr_ipw_classes;

typedef struct {
  bsr_choose_fn inner;
  bsr_assumed_fn inner_assumed;   /* may be NULL */
  void* inner_ctx;
  uint32_t n_nodes;
  const uint32_t* topo;           /* [n_keys][n_nodes] */
  const uint32_t* term_key;       /* [n_terms] */
  uint32_t n_bound;
  const uint32_t* bound_node;     /* [n_bound] */
  const uint32_t* bound_class;    /* [n_bound] */
  bsr_ipw_classes bound;          /* (term, own, match) */
  const uint32_t* pod_class;      /* [n_pods] filter class */
  const uint32_t* p_off;          /* filter classes: (term, role), self_match */
  const uint32_t* p_term;
  const uint8_t* p_role;
  const uint8_t* p_self;
  const uint32_t* placed_class;   /* [n_pods] */
  bsr_ipw_classes placed;         /* (term, own, match) */
  uint32_t* assumed_pod;          /* [capacity] the walk's assumed pods so far, in order */
  uint32_t* assumed_node;
  uint32_t n_assumed;
} bsr_ipw_ctx;

static uint32_t value(const bsr_ipw_ctx* c, uint32_t t, uint32_t node) {
  return c->topo[(size_t)c->term_key[t] * c->n_nodes + node];
}

/* does class `cls` of table `tab` list term t with own (want_own) or match set? */
static int class_has(const bsr_ipw_classes* tab, uint32_t cls, uint32_t t, int want_own) {
  if (cls == BSR_IPW_NONE) return 0;
  for (uint32_t k = tab->off[cls]; k < tab->off[cls + 1]; ++k)
    if (tab->term[k] == t) return want_own ? tab->own[k] != 0 : tab->match[k] != 0;
  return 0;
}

/* existing pod e: the bound pods first, then the assumed ones */
static uint32_t existing_count(const bsr_ipw_ctx* c) { return c->n_bound + c->n_assumed; }
static uint32_t existing_node(const bsr_ipw_ctx* c, uint32_t e) {
  return e < c->n_bound ? c->bound_node[e] : c->assumed_node[e - c->n_bound];
}
static int existing_has(const bsr_ipw_ctx* c, uint32_t e, uint32_t t, int want_own) {
  if (e < c->n_bound) return class_has(&c->bound, c->bound_class[e], t, want_own);
  return class_has(&c->placed, c->placed_class[c->assumed_pod[e - c->n_bound]], t, want_own);
}

/* some existing pod with own / match on t sits on a node whose value of key(t) is v */
static int some_existing(const bsr_ipw_ctx* c, uint32_t t, uint32_t v, int want_own) {
  for (uint32_t e = 0; e < existing_count(c); ++e)
    if (existing_has(c, e, t, want_own) && value(c, t, existing_node(c, e)) == v) return 1;
  return 0;
}

/* step 1 for one term w: n carries key(w) and an existing pod owning w sits in n's topology */
static int fails_existing(const bsr_ipw_ctx* c, uint32_t w, uint32_t n) {
  const uint32_t v = value(c, w, n);
  return v != BSR_IPW_TOPO_NONE && some_existing(c, w, v, 1);
}

/* 1 when pod p passes node n against the bound and the assumed pods */
int bsr_ipw_pass(const bsr_ipw_ctx* c, uint32_t p, uint32_t n) {
  const uint32_t fc = c->pod_class[p], qc = c->placed_class[p];
  /* 1. existing pods' anti-affinity: the filter class's EXISTING entries and the placed class's match entries */
  if (fc != BSR_IPW_NONE)
    for (uint32_t k = c->p_off[fc]; k < c->p_off[fc + 1]; ++k)
      if (c->p_role[k] == BSR_IPW_EXISTING && fails_existing(c, c->p_term[k], n)) return 0;
  if (qc != BSR_IPW_NONE)
    for (uint32_t k = c->placed.off[qc]; k < c->placed.off[qc + 1]; ++k)
      if (c->placed.match[k] && fails_existing(c, c->placed.term[k], n)) return 0;
  if (fc == BSR_IPW_NONE) return 1;
  const uint32_t o0 = c->p_off[fc], o1 = c->p_off[fc + 1];
  /* 2. no affinity of its own */
  int n_aff = 0, n_anti = 0;
  for (uint32_t k = o0; k < o1; ++k) {
    n_aff += c->p_role[k] == BSR_IPW_AFFINITY;
    n_anti += c->p_role[k] == BSR_IPW_ANTI;
  }
  if (!n_aff && !n_anti) return 1;
  /* 3. affinity: every term has a matching pod in n's topology, or the first-pod exception */
  if (n_aff) {
    int all = 1, any_pair = 0;
    for (uint32_t k = o0; k < o1; ++k) {
      if (c->p_role[k] != BSR_IPW_AFFINITY) continue;
      const uint32_t t = c->p_term[k], v = value(c, t, n);
      if (v == BSR_IPW_TOPO_NONE || !some_existing(c, t, v, 0)) all = 0;
      for (uint32_t e = 0; e < existing_count(c); ++e)
        if (existing_has(c, e, t, 0) && value(c, t, existing_node(c, e)) != BSR_IPW_TOPO_NONE) any_pair = 1;
    }
    if (!all && !(!any_pair && c->p_self[fc])) return 0;
  }
  /* 4. anti-affinity */
  for (uint32_t k = o0; k < o1; ++k) {
    if (c->p_role[k] != BSR_IPW_ANTI) continue;
    const uint32_t v = value(c, c->p_term[k], n);
    if (v != BSR_IPW_TOPO_NONE && some_existing(c, c->p_term[k], v, 0)) return 0;
  }
  return 1;
}

/* The wrapped chooser over the nodes that pass: the others are flagged unschedulable while it runs, so that
 * bso_fit_eval skips them, and get their flags back before the walk goes on. */
int32_t bsr_ipw_choose(void* ctx, const bso_nodes* nd, const bso_pods* pd, uint32_t p) {
  const bsr_ipw_ctx* c = (const bsr_ipw_ctx*)ctx;
  uint8_t* saved = (uint8_t*)malloc(nd->n ? nd->n : 1);
  for (uint32_t n = 0; n < nd->n; ++n) {
    saved[n] = nd->flags[n];
    if (!bsr_ipw_pass(c, p, n)) nd->flags[n] |= BSO_NODE_UNSCHEDULABLE;
  }
  const int32_t r = c->inner(c->inner_ctx, nd, pd, p);
  for (uint32_t n = 0; n < nd->n; ++n) nd->flags[n] = saved[n];
  free(saved);
  return r;
}

/* NodeInfo.AddPod: the pod joins the existing pods of node n with its placed class */
void bsr_ipw_assumed(void* ctx, const bso_nodes* nd, const bso_pods* pd, uint32_t p, uint32_t n) {
  bsr_ipw_ctx* c = (bsr_ipw_ctx*)ctx;
  c->assumed_pod[c->n_assumed] = p;
  c->assumed_node[c->n_assumed] = n;
  c->n_assumed++;
  if (c->inner_assumed) c->inner_assumed(c->inner_ctx, nd, pd, p, n);
}
