/* ratio_priority_ref.c — TEST INFRASTRUCTURE: the CPU restatement of kube-scheduler v1.17's RequestedToCapacityRatio
 * priority as the engine adds it to the resource priorities (include/bsched.h bs_set_ratio_priority), written from
 * requested_to_capacity_ratio.go and resource_allocation.go [upstream, from memory].  The shape is evaluated straight
 * from the broken-line definition at each utilization, not from a table, and the average is rounded with C's round()
 * (half away from zero, Go's math.Round) on binary64.  The score is bsr_priority_score (tests/priority_ref.c) plus
 * weight * Ratio.  Provides the priority-list builder over bso_fit_eval and a chooser / assume hook pair for
 * bsr_replay_choose (tests/replay_priority_ref.c).  Compiled with -ffp-contract=off; tests/ratio_priority_ref.py
 * compiles it with both files into a temporary directory and binds it. */
#include <math.h>
#include <stddef.h>
#include <stdint.h>

#include "bs_oracle.h"

int64_t bsr_priority_score(int64_t r_cpu, int64_t c_cpu, int64_t r_mem, int64_t c_mem, uint32_t w_least, uint32_t w_most,
                           uint32_t w_balanced);
typedef int32_t (*bsr_choose_fn)(void* ctx, const bso_nodes* nd, const bso_pods* pd, uint32_t p);
typedef void (*bsr_assumed_fn)(void* ctx, const bso_nodes* nd, const bso_pods* pd, uint32_t p, uint32_t n);
int bsr_replay_choose(bso_nodes* nd, const bso_pods* pd, bso_groups* gr, const uint32_t* queue, uint32_t n_queue,
                      uint8_t* prefilter_out, int32_t* node_out, uint8_t* ready_out, bsr_choose_fn choose,
                      bsr_assumed_fn assumed, void* ctx);

/* the setting of bs_set_ratio_priority, in engine units */
typedef struct {
  uint32_t weight, n_points;
  int64_t utilization[101], score[101];
  uint32_t n_lanes;
  uint32_t lane_weight[BSO_MAX_LANES];
  uint32_t absent_weight;
} bsr_ratio_setting;

/* buildBrokenLinearFunction: s_0 at or below the first point, the last score above the last point, else the segment
 * u_{i-1} < p <= u_i, int64 truncating toward zero */
int64_t bsr_ratio_shape(const bsr_ratio_setting* s, int64_t p) {
  for (uint32_t i = 0; i < s->n_points; ++i) {
    if (p > s->utilization[i]) continue;
    if (i == 0) return s->score[0];
    return s->score[i - 1] + (s->score[i] - s->score[i - 1]) * (p - s->utilization[i - 1]) /
                                 (s->utilization[i] - s->utilization[i - 1]);
  }
  return s->score[s->n_points - 1];
}

/* maxUtilization - (capacity - requested) * maxUtilization / capacity, 100 when capacity is 0 or exceeded; Go's int64
 * wraps, so the differences and the product are taken unsigned, and MinInt64 / -1 is MinInt64 */
int64_t bsr_ratio_util(int64_t r, int64_t c) {
  if (c == 0 || r > c) return 100;
  const int64_t prod = (int64_t)(((uint64_t)c - (uint64_t)r) * 100u);
  const int64_t q = (c == -1) ? (int64_t)(0 - (uint64_t)prod) : prod / c;
  return (int64_t)(100u - (uint64_t)q);
}

/* Ratio from the per-lane requested r[d] and capacity c[d] (a missing key already 0): the weighted average of the
 * resources that score above 0, the resources no node has joining with shape(100) */
int64_t bsr_ratio_of(const bsr_ratio_setting* s, const int64_t* r, const int64_t* c) {
  int64_t num = 0, den = 0;
  for (uint32_t d = 0; d < s->n_lanes; ++d) {
    if (!s->lane_weight[d]) continue;
    const int64_t sc = bsr_ratio_shape(s, bsr_ratio_util(r[d], c[d]));
    if (sc > 0) { num += sc * s->lane_weight[d]; den += s->lane_weight[d]; }
  }
  const int64_t full = bsr_ratio_shape(s, 100);
  if (full > 0 && s->absent_weight) { num += full * s->absent_weight; den += s->absent_weight; }
  if (den == 0) return 0;
  return (int64_t)round((double)num / (double)den);
}

/* Ratio of pod p on node n: cpu and memory from the non-zero columns, lane 2 and the scalar lanes from the node table's
 * (live) requested plus the pod table's request, a key absent on a side counting 0 there */
int64_t bsr_ratio_pair(const bsr_ratio_setting* s, const bso_nodes* nd, const bso_pods* pd, const int64_t* node_nz,
                       const int64_t* pod_nz, uint32_t p, uint32_t n) {
  const uint32_t N = nd->n, P = pd->n;
  int64_t r[BSO_MAX_LANES] = {0}, c[BSO_MAX_LANES] = {0};
  for (uint32_t d = 0; d < s->n_lanes; ++d) {
    if (d < 2) {
      r[d] = node_nz[(size_t)d * N + n] + pod_nz[(size_t)d * P + p];
      c[d] = nd->alloc[(size_t)d * N + n];
      continue;
    }
    const uint32_t bit = 1u << d;
    const int fixed = d < 4;
    const int64_t rn = (fixed || (nd->req_present[n] & bit)) ? nd->requested[(size_t)d * N + n] : 0;
    const int64_t rp = (fixed || (pd->req_present[p] & bit)) ? pd->req[(size_t)d * P + p] : 0;
    r[d] = (int64_t)((uint64_t)rn + (uint64_t)rp);
    c[d] = (fixed || (nd->alloc_present[n] & bit)) ? nd->alloc[(size_t)d * N + n] : 0;
  }
  return bsr_ratio_of(s, r, c);
}

/* the whole score: the three resource priorities plus weight * Ratio, int64 wrapping */
int64_t bsr_ratio_total(const bsr_ratio_setting* s, const bso_nodes* nd, const bso_pods* pd, const int64_t* node_nz,
                        const int64_t* pod_nz, uint32_t p, uint32_t n, uint32_t w_least, uint32_t w_most,
                        uint32_t w_balanced) {
  const uint32_t N = nd->n, P = pd->n;
  const int64_t base = bsr_priority_score(node_nz[n] + pod_nz[p], nd->alloc[n], node_nz[(size_t)N + n] + pod_nz[(size_t)P + p],
                                          nd->alloc[(size_t)N + n], w_least, w_most, w_balanced);
  if (!s->weight) return base;
  return (int64_t)((uint64_t)base + (uint64_t)s->weight * (uint64_t)bsr_ratio_pair(s, nd, pd, node_nz, pod_nz, p, n));
}

/* The list of pod p (as bsr_priority_rows): its fitting nodes by the whole score descending, then node index ascending,
 * the first K, padded with node -1 and score INT64_MIN */
void bsr_ratio_rows(const bsr_ratio_setting* s, const bso_nodes* nd, const bso_pods* pd, const int64_t* node_nz,
                    const int64_t* pod_nz, uint32_t p, uint32_t K, uint32_t w_least, uint32_t w_most, uint32_t w_balanced,
                    int32_t* nodes, int64_t* scores) {
  uint32_t filled = 0;
  for (uint32_t k = 0; k < K; ++k) { nodes[k] = -1; scores[k] = INT64_MIN; }
  for (uint32_t n = 0; n < nd->n; ++n) {
    if (!bso_fit_eval(nd, pd, p, n, NULL)) continue;
    const int64_t sc = bsr_ratio_total(s, nd, pd, node_nz, pod_nz, p, n, w_least, w_most, w_balanced);
    uint32_t pos = 0;
    while (pos < filled && scores[pos] >= sc) ++pos;
    if (pos >= K) continue;
    for (uint32_t k = (filled < K ? filled : K - 1); k > pos; --k) { nodes[k] = nodes[k - 1]; scores[k] = scores[k - 1]; }
    nodes[pos] = (int32_t)n;
    scores[pos] = sc;
    if (filled < K) ++filled;
  }
}

/* The chooser / assume hooks for bsr_replay_choose: the live node column node_nz grows on every assume; `requested`
 * and req_present are the walk's live tables */
typedef struct {
  int64_t* node_nz;
  const int64_t* pod_nz;
  uint32_t w_least, w_most, w_balanced;
  const bsr_ratio_setting* s;
} bsr_ratio_ctx;

int32_t bsr_ratio_choose(void* ctx, const bso_nodes* nd, const bso_pods* pd, uint32_t p) {
  const bsr_ratio_ctx* c = (const bsr_ratio_ctx*)ctx;
  int32_t best = -1;
  int64_t best_s = INT64_MIN;
  for (uint32_t n = 0; n < nd->n; ++n) {
    if (!bso_fit_eval(nd, pd, p, n, NULL)) continue;
    const int64_t sc = bsr_ratio_total(c->s, nd, pd, c->node_nz, c->pod_nz, p, n, c->w_least, c->w_most, c->w_balanced);
    if (best < 0 || sc > best_s) { best = (int32_t)n; best_s = sc; }   /* ascending nodes: ties keep the lower index */
  }
  return best;
}

void bsr_ratio_assumed(void* ctx, const bso_nodes* nd, const bso_pods* pd, uint32_t p, uint32_t n) {
  bsr_ratio_ctx* c = (bsr_ratio_ctx*)ctx;
  c->node_nz[n] += c->pod_nz[p];
  c->node_nz[(size_t)nd->n + n] += c->pod_nz[(size_t)pd->n + p];
}

/* bs_replay_priority with the ratio term: node_nz [2][n_nodes] is the live column, updated in place */
int bsr_replay_ratio(bso_nodes* nd, const bso_pods* pd, bso_groups* gr, const uint32_t* queue, uint32_t n_queue,
                     uint8_t* prefilter_out, int32_t* node_out, uint8_t* ready_out, int64_t* node_nz, const int64_t* pod_nz,
                     uint32_t w_least, uint32_t w_most, uint32_t w_balanced, const bsr_ratio_setting* s) {
  bsr_ratio_ctx c = {node_nz, pod_nz, w_least, w_most, w_balanced, s};
  return bsr_replay_choose(nd, pd, gr, queue, n_queue, prefilter_out, node_out, ready_out, bsr_ratio_choose,
                           bsr_ratio_assumed, &c);
}
