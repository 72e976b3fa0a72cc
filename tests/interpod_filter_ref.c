/* interpod_filter_ref.c — TEST INFRASTRUCTURE: the CPU restatement of kube-scheduler v1.17's MatchInterPodAffinity
 * filter as the engine applies it (include/bsched.h bs_set_interpod_filter), on the packed columns of
 * bs_upload_node_interpod_filter / bs_upload_pod_interpod_filter.  No presence tables: for each (pod, node) it loops
 * over the bound pods directly, in the order of the four steps, and returns the step that failed.
 * tests/interpod_filter_ref.py compiles it into a library of its own. */
#include <stddef.h>
#include <stdint.h>

#define BSR_IPF_NONE 0xffffffffu
#define BSR_TOPO_NONE 0xffffffffu
enum { BSR_AFFINITY = 0, BSR_ANTI = 1, BSR_EXISTING = 2 };
enum { BSR_PASS = 0, BSR_FAIL_E = 1, BSR_FAIL_A = 2, BSR_FAIL_N = 3 };

typedef struct {
  uint32_t n_nodes;
  const uint32_t* topo;        /* [n_keys][n_nodes] */
  const uint32_t* term_key;    /* [n_terms] */
  uint32_t n_bound;
  const uint32_t* bound_node;  /* [n_bound] */
  const uint32_t* bound_class; /* [n_bound] */
  const uint32_t* b_off;       /* bound classes: (term, own, match) */
  const uint32_t* b_term;
  const int32_t* b_own;
  const uint8_t* b_match;
  const uint32_t* pod_class;   /* [n_pods] */
  const uint32_t* p_off;       /* pod classes: (term, role), self_match */
  const uint32_t* p_term;
  const uint8_t* p_role;
  const uint8_t* p_self;
} bsr_ipf;

static uint32_t value(const bsr_ipf* q, uint32_t t, uint32_t node) {
  return q->topo[(size_t)q->term_key[t] * q->n_nodes + node];
}

/* does bound pod e list term t with own (want_own) or match set? */
static int bound_has(const bsr_ipf* q, uint32_t e, uint32_t t, int want_own) {
  const uint32_t c = q->bound_class[e];
  if (c == BSR_IPF_NONE) return 0;
  for (uint32_t k = q->b_off[c]; k < q->b_off[c + 1]; ++k)
    if (q->b_term[k] == t) return want_own ? q->b_own[k] != 0 : q->b_match[k] != 0;
  return 0;
}

/* some bound pod with own / match on t sits on a node whose value of key(t) is v */
static int some_bound(const bsr_ipf* q, uint32_t t, uint32_t v, int want_own) {
  for (uint32_t e = 0; e < q->n_bound; ++e)
    if (bound_has(q, e, t, want_own) && value(q, t, q->bound_node[e]) == v) return 1;
  return 0;
}

int bsr_ipf_verdict(const bsr_ipf* q, uint32_t p, uint32_t n) {
  const uint32_t c = q->pod_class[p];
  if (c == BSR_IPF_NONE) return BSR_PASS;
  const uint32_t o0 = q->p_off[c], o1 = q->p_off[c + 1];
  /* 1. existing pods' anti-affinity */
  for (uint32_t k = o0; k < o1; ++k) {
    if (q->p_role[k] != BSR_EXISTING) continue;
    const uint32_t v = value(q, q->p_term[k], n);
    if (v != BSR_TOPO_NONE && some_bound(q, q->p_term[k], v, 1)) return BSR_FAIL_E;
  }
  /* 2. no affinity of its own */
  int n_aff = 0, n_anti = 0;
  for (uint32_t k = o0; k < o1; ++k) {
    n_aff += q->p_role[k] == BSR_AFFINITY;
    n_anti += q->p_role[k] == BSR_ANTI;
  }
  if (!n_aff && !n_anti) return BSR_PASS;
  /* 3. affinity: every term has a matching pod in n's topology, or the first-pod exception */
  if (n_aff) {
    int all = 1, any_pair = 0;
    for (uint32_t k = o0; k < o1; ++k) {
      if (q->p_role[k] != BSR_AFFINITY) continue;
      const uint32_t t = q->p_term[k], v = value(q, t, n);
      if (v == BSR_TOPO_NONE || !some_bound(q, t, v, 0)) all = 0;
      for (uint32_t e = 0; e < q->n_bound; ++e)
        if (bound_has(q, e, t, 0) && value(q, t, q->bound_node[e]) != BSR_TOPO_NONE) any_pair = 1;
    }
    if (!all && !(!any_pair && q->p_self[c])) return BSR_FAIL_A;
  }
  /* 4. anti-affinity */
  for (uint32_t k = o0; k < o1; ++k) {
    if (q->p_role[k] != BSR_ANTI) continue;
    const uint32_t v = value(q, q->p_term[k], n);
    if (v != BSR_TOPO_NONE && some_bound(q, q->p_term[k], v, 0)) return BSR_FAIL_N;
  }
  return BSR_PASS;
}

/* out[k * n_nodes + n] = the verdict of pods[k] on node n */
void bsr_ipf_matrix(const bsr_ipf* q, const uint32_t* pods, uint32_t n_pods, uint8_t* out) {
  for (uint32_t k = 0; k < n_pods; ++k)
    for (uint32_t n = 0; n < q->n_nodes; ++n) out[(size_t)k * q->n_nodes + n] = (uint8_t)bsr_ipf_verdict(q, pods[k], n);
}
