/* interpod_priority_ref.c — TEST INFRASTRUCTURE: the CPU restatement of kube-scheduler v1.17's InterPodAffinity
 * priority as the engine adds it to the priority lists (include/bsched.h bs_set_interpod_weight), written from
 * interpod_affinity.go [upstream, from memory] on the packed columns of bs_upload_node_interpod /
 * bs_upload_pod_interpod.  The raw score of a pod is computed as upstream computes it, not through the engine's term x
 * value tables: for every bound pod e and every term both classes list, the weight that term adds (p's own weight if
 * e matches it, e's own weight if p matches it) goes to topologyScore[key][value of key on e's node]; each node then
 * sums the entries of its own values.  The reduce runs over the pod's fit set as upstream runs over the filtered nodes,
 * with both extremes started at 0.  The rest of the score is tests/spread_priority_ref.c's (the resource score, and
 * when given the node, locality and spread terms), so every flag combination of the lists has a restatement.
 * tests/interpod_priority_ref.py compiles it with -ffp-contract=off into a library of its own. */
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "bs_oracle.h"

#define BSR_IPA_NONE 0xffffffffu
#define BSR_TOPO_NONE 0xffffffffu

/* tests/ratio_priority_ref.c */
int64_t bsr_ratio_total(const void* setting, const bso_nodes* nd, const bso_pods* pd, const int64_t* node_nz,
                        const int64_t* pod_nz, uint32_t p, uint32_t n, uint32_t w_least, uint32_t w_most,
                        uint32_t w_balanced);

/* tests/node_priority_ref.c */
typedef struct {
  const uint64_t* prefer_taints;
  const int32_t* pref_weights;
  const uint64_t* prefer_tol;
  const uint32_t* pref_class;
  uint32_t w_taint, w_naff;
} bsr_node_pref;
int64_t bsr_taint_raw(const bsr_node_pref* q, uint32_t p, uint32_t n);
int64_t bsr_naff_raw(const bsr_node_pref* q, const bso_nodes* nd, uint32_t p, uint32_t n);
int64_t bsr_normalize(int64_t raw, int64_t mx, int reverse);
void bsr_node_pref_maxima(const bsr_node_pref* q, const bso_nodes* nd, const bso_pods* pd, uint32_t p, int64_t* mt,
                          int64_t* ma);

/* tests/locality_priority_ref.c */
uint64_t bsr_locality_term(const void* q, const bso_nodes* nd, uint32_t p, uint32_t n);

/* tests/spread_priority_ref.c: its columns stay opaque here except the weight, its last field */
typedef struct {
  const void* zone;
  const void* counts;
  const void* spread_class;
  uint32_t w_spread;
} bsr_spread;
void bsr_spread_reduce(const bsr_spread* q, const bso_nodes* nd, const bso_pods* pd, uint32_t p, int64_t* ss);

/* the columns of bs_upload_node_interpod / bs_upload_pod_interpod and the weight */
typedef struct {
  uint32_t n_keys;
  const uint32_t* n_values;      /* [n_keys] */
  const uint32_t* topo;          /* [n_keys][n_nodes] */
  uint32_t n_terms;
  const uint32_t* term_key;      /* [n_terms] */
  uint32_t n_bound;
  const uint32_t* bound_node;    /* [n_bound] */
  const uint32_t* bound_class;   /* [n_bound] */
  const uint32_t* b_off;         /* the bound classes */
  const uint32_t* b_term;
  const int32_t* b_own;
  const uint8_t* b_match;
  const uint32_t* pod_class;     /* [n_pods] */
  const uint32_t* p_off;         /* the pod classes */
  const uint32_t* p_term;
  const int32_t* p_own;
  const uint8_t* p_match;
  uint32_t w_ipa;
} bsr_ipa;

/* raw[n] of pod p on every node (0 for a pod without a class) */
void bsr_ipa_raw(const bsr_ipa* q, uint32_t n_nodes, uint32_t p, int64_t* raw) {
  memset(raw, 0, (size_t)n_nodes * sizeof(int64_t));
  const uint32_t c = q->pod_class[p];
  if (c == BSR_IPA_NONE) return;
  size_t total = 0;
  size_t* base = (size_t*)malloc((q->n_keys + 1) * sizeof(size_t));
  for (uint32_t k = 0; k < q->n_keys; ++k) { base[k] = total; total += q->n_values[k]; }
  int64_t* topology_score = (int64_t*)calloc(total ? total : 1, sizeof(int64_t));
  /* the pod's entry of each term (-1: none) */
  int64_t* entry_of = (int64_t*)malloc((q->n_terms ? q->n_terms : 1) * sizeof(int64_t));
  for (uint32_t t = 0; t < q->n_terms; ++t) entry_of[t] = -1;
  for (uint32_t a = q->p_off[c]; a < q->p_off[c + 1]; ++a) entry_of[q->p_term[a]] = a;
  for (uint32_t e = 0; e < q->n_bound; ++e) {
    const uint32_t ce = q->bound_class[e];
    if (ce == BSR_IPA_NONE) continue;
    for (uint32_t b = q->b_off[ce]; b < q->b_off[ce + 1]; ++b) {
      if (entry_of[q->b_term[b]] < 0) continue;
      const uint32_t a = (uint32_t)entry_of[q->b_term[b]];
      const uint32_t key = q->term_key[q->p_term[a]];
      const uint32_t v = q->topo[(size_t)key * n_nodes + q->bound_node[e]];
      if (v == BSR_TOPO_NONE) continue;   /* e's node lacks the key: no node shares its value */
      /* p's own terms checked against e, then e's own terms checked against p */
      topology_score[base[key] + v] += (int64_t)q->p_own[a] * q->b_match[b] + (int64_t)q->b_own[b] * q->p_match[a];
    }
  }
  for (uint32_t n = 0; n < n_nodes; ++n)
    for (uint32_t k = 0; k < q->n_keys; ++k) {
      const uint32_t v = q->topo[(size_t)k * n_nodes + n];
      if (v != BSR_TOPO_NONE) raw[n] += topology_score[base[k] + v];
    }
  free(topology_score);
  free(entry_of);
  free(base);
}

/* the reduce of one node: binary64, each operation rounded on its own (-ffp-contract=off), truncation toward zero */
int64_t bsr_ipa_score(int64_t raw, int64_t mn, int64_t mx) {
  double f = 0.0;
  if (mx - mn > 0) f = 100.0 * ((double)(raw - mn) / (double)(mx - mn));
  return (int64_t)f;
}

/* CalculateInterPodAffinityPriorityReduce over the fit set of pod p: ipa[n] for every fitting node (others
 * untouched) */
void bsr_ipa_reduce(const bsr_ipa* q, const bso_nodes* nd, const bso_pods* pd, uint32_t p, int64_t* ipa) {
  int64_t* raw = (int64_t*)malloc((nd->n ? nd->n : 1) * sizeof(int64_t));
  bsr_ipa_raw(q, nd->n, p, raw);
  int64_t mn = 0, mx = 0;
  for (uint32_t n = 0; n < nd->n; ++n) {
    if (!bso_fit_eval(nd, pd, p, n, NULL)) continue;
    if (raw[n] > mx) mx = raw[n];
    if (raw[n] < mn) mn = raw[n];
  }
  for (uint32_t n = 0; n < nd->n; ++n)
    if (bso_fit_eval(nd, pd, p, n, NULL)) ipa[n] = bsr_ipa_score(raw[n], mn, mx);
  free(raw);
}

/* The list of pod p (as bsr_spread_rows): its fitting nodes by the whole score descending, then node index ascending,
 * the first K, padded with node -1 and score INT64_MIN.  pref, loc, spread: the other priorities' columns (NULL: off). */
void bsr_interpod_rows(const bsr_ipa* q, const bsr_spread* spread, const bsr_node_pref* pref, const void* loc,
                       const void* s, const bso_nodes* nd, const bso_pods* pd, const int64_t* node_nz,
                       const int64_t* pod_nz, uint32_t p, uint32_t K, uint32_t w_least, uint32_t w_most,
                       uint32_t w_balanced, int32_t* nodes, int64_t* scores) {
  int64_t mt = 0, ma = 0;
  if (pref) bsr_node_pref_maxima(pref, nd, pd, p, &mt, &ma);
  int64_t* ss = (int64_t*)calloc(nd->n ? nd->n : 1, sizeof(int64_t));
  int64_t* ipa = (int64_t*)calloc(nd->n ? nd->n : 1, sizeof(int64_t));
  if (spread && spread->w_spread) bsr_spread_reduce(spread, nd, pd, p, ss);
  if (q->w_ipa) bsr_ipa_reduce(q, nd, pd, p, ipa);
  uint32_t filled = 0;
  for (uint32_t k = 0; k < K; ++k) { nodes[k] = -1; scores[k] = INT64_MIN; }
  for (uint32_t n = 0; n < nd->n; ++n) {
    if (!bso_fit_eval(nd, pd, p, n, NULL)) continue;
    uint64_t sc = (uint64_t)bsr_ratio_total(s, nd, pd, node_nz, pod_nz, p, n, w_least, w_most, w_balanced);
    if (pref) {
      const int64_t tt = bsr_normalize(pref->w_taint ? bsr_taint_raw(pref, p, n) : 0, mt, 1);
      const int64_t na = bsr_normalize(pref->w_naff ? bsr_naff_raw(pref, nd, p, n) : 0, ma, 0);
      sc += (uint64_t)pref->w_taint * (uint64_t)tt + (uint64_t)pref->w_naff * (uint64_t)na;
    }
    if (loc) sc += bsr_locality_term(loc, nd, p, n);
    if (spread) sc += (uint64_t)spread->w_spread * (uint64_t)ss[n];
    sc += (uint64_t)q->w_ipa * (uint64_t)ipa[n];
    const int64_t v = (int64_t)sc;
    uint32_t pos = 0;
    while (pos < filled && scores[pos] >= v) ++pos;
    if (pos >= K) continue;
    for (uint32_t k = (filled < K ? filled : K - 1); k > pos; --k) { nodes[k] = nodes[k - 1]; scores[k] = scores[k - 1]; }
    nodes[pos] = (int32_t)n;
    scores[pos] = v;
    if (filled < K) ++filled;
  }
  free(ss);
  free(ipa);
}
