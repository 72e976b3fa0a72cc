/* node_priority_ref.c — TEST INFRASTRUCTURE: the CPU restatement of kube-scheduler v1.17's TaintToleration and
 * preferred NodeAffinity priorities as the engine adds them to the resource priorities (include/bsched.h
 * bs_set_node_priority_weights), written from taint_toleration.go, node_affinity.go and DefaultNormalizeScore
 * [upstream, from memory].  Each pod's two maxima are taken over its fit set (the oracle's bso_fit_eval) before any
 * node is scored; the resource part of the score is bsr_ratio_total (tests/ratio_priority_ref.c), so the ratio term
 * joins with a non-zero weight in its setting.  tests/node_priority_ref.py compiles it with -ffp-contract=off into a
 * library of its own, linked against tests/native.py's library of the other restatements, and binds it. */
#include <stddef.h>
#include <stdint.h>

#include "bs_oracle.h"

#define BSR_PREF_NONE 0xffffffffu

/* tests/ratio_priority_ref.c, reached through tests/native.py's library: the whole resource score of pod p on node n
 * (bsr_priority_score plus weight * Ratio).  Its setting is built by tests/ratio_priority_ref.py and only passed
 * through here, so its layout stays private to that file. */
int64_t bsr_ratio_total(const void* setting, const bso_nodes* nd, const bso_pods* pd, const int64_t* node_nz,
                        const int64_t* pod_nz, uint32_t p, uint32_t n, uint32_t w_least, uint32_t w_most,
                        uint32_t w_balanced);

/* the columns of bs_upload_node_preferences / bs_upload_pod_preferences and the two weights */
typedef struct {
  const uint64_t* prefer_taints;   /* [n_nodes] */
  const int32_t* pref_weights;     /* [n_classes][n_nodes] */
  const uint64_t* prefer_tol;      /* [n_pods] */
  const uint32_t* pref_class;      /* [n_pods] */
  uint32_t w_taint, w_naff;
} bsr_node_pref;

static int64_t popcount64(uint64_t x) {
  int64_t c = 0;
  for (; x; x &= x - 1) ++c;
  return c;
}

/* raw TaintToleration count: the node's PreferNoSchedule taints the pod does not tolerate */
int64_t bsr_taint_raw(const bsr_node_pref* q, uint32_t p, uint32_t n) {
  return popcount64(q->prefer_taints[n] & ~q->prefer_tol[p]);
}

/* raw NodeAffinity count: the summed weights of the pod's preferred terms the node matches */
int64_t bsr_naff_raw(const bsr_node_pref* q, const bso_nodes* nd, uint32_t p, uint32_t n) {
  const uint32_t c = q->pref_class[p];
  return c == BSR_PREF_NONE ? 0 : q->pref_weights[(size_t)c * nd->n + n];
}

/* NormalizeReduce(100, reverse) of one raw count against the maximum */
int64_t bsr_normalize(int64_t raw, int64_t mx, int reverse) {
  if (mx == 0) return reverse ? 100 : 0;
  const int64_t s = 100 * raw / mx;
  return reverse ? 100 - s : s;
}

/* the maxima of pod p's raw counts over the nodes where it fits; mt, ma stay 0 when none does */
void bsr_node_pref_maxima(const bsr_node_pref* q, const bso_nodes* nd, const bso_pods* pd, uint32_t p, int64_t* mt,
                          int64_t* ma) {
  *mt = *ma = 0;
  for (uint32_t n = 0; n < nd->n; ++n) {
    if (!bso_fit_eval(nd, pd, p, n, NULL)) continue;
    const int64_t t = bsr_taint_raw(q, p, n), a = bsr_naff_raw(q, nd, p, n);
    if (t > *mt) *mt = t;
    if (a > *ma) *ma = a;
  }
}

/* The list of pod p (as bsr_priority_rows): its fitting nodes by the whole score descending, then node index
 * ascending, the first K, padded with node -1 and score INT64_MIN.  s: the ratio setting (weight 0 = no ratio term). */
void bsr_node_priority_rows(const bsr_node_pref* q, const void* s, const bso_nodes* nd, const bso_pods* pd,
                            const int64_t* node_nz, const int64_t* pod_nz, uint32_t p, uint32_t K, uint32_t w_least,
                            uint32_t w_most, uint32_t w_balanced, int32_t* nodes, int64_t* scores) {
  int64_t mt, ma;
  bsr_node_pref_maxima(q, nd, pd, p, &mt, &ma);
  uint32_t filled = 0;
  for (uint32_t k = 0; k < K; ++k) { nodes[k] = -1; scores[k] = INT64_MIN; }
  for (uint32_t n = 0; n < nd->n; ++n) {
    if (!bso_fit_eval(nd, pd, p, n, NULL)) continue;
    const int64_t tt = bsr_normalize(bsr_taint_raw(q, p, n), mt, 1);
    const int64_t na = bsr_normalize(bsr_naff_raw(q, nd, p, n), ma, 0);
    const uint64_t base = (uint64_t)bsr_ratio_total(s, nd, pd, node_nz, pod_nz, p, n, w_least, w_most, w_balanced);
    const int64_t sc = (int64_t)(base + (uint64_t)q->w_taint * (uint64_t)tt + (uint64_t)q->w_naff * (uint64_t)na);
    uint32_t pos = 0;
    while (pos < filled && scores[pos] >= sc) ++pos;
    if (pos >= K) continue;
    for (uint32_t k = (filled < K ? filled : K - 1); k > pos; --k) { nodes[k] = nodes[k - 1]; scores[k] = scores[k - 1]; }
    nodes[pos] = (int32_t)n;
    scores[pos] = sc;
    if (filled < K) ++filled;
  }
}
