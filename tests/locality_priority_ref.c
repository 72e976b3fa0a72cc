/* locality_priority_ref.c — TEST INFRASTRUCTURE: the CPU restatement of kube-scheduler v1.17's ImageLocality and
 * NodePreferAvoidPods priorities as the engine adds them to the priority lists and to bs_replay_priority's node choice
 * (include/bsched.h bs_set_locality_weights), written from image_locality.go and node_prefer_avoid_pods.go [upstream,
 * from memory].  Both terms are static per (pod, node), so nothing here looks at the fit set beyond choosing the nodes
 * that are scored.  The rest of the score is tests/ratio_priority_ref.c's bsr_ratio_total plus, in the lists, the
 * TaintToleration and NodeAffinity terms of tests/node_priority_ref.c.  tests/locality_priority_ref.py compiles it
 * with -ffp-contract=off into a library of its own, linked against both of those libraries and the oracle. */
#include <stddef.h>
#include <stdint.h>

#include "bs_oracle.h"

#define BSR_IMAGE_NONE 0xffffffffu
#define BSR_AVOID_NONE 0xffu
#define BSR_MIB ((int64_t)1 << 20)

/* tests/ratio_priority_ref.c and tests/replay_priority_ref.c (tests/native.py's library) */
int64_t bsr_ratio_total(const void* setting, const bso_nodes* nd, const bso_pods* pd, const int64_t* node_nz,
                        const int64_t* pod_nz, uint32_t p, uint32_t n, uint32_t w_least, uint32_t w_most,
                        uint32_t w_balanced);
typedef int32_t (*bsr_choose_fn)(void* ctx, const bso_nodes* nd, const bso_pods* pd, uint32_t p);
typedef void (*bsr_assumed_fn)(void* ctx, const bso_nodes* nd, const bso_pods* pd, uint32_t p, uint32_t n);
int bsr_replay_choose(bso_nodes* nd, const bso_pods* pd, bso_groups* gr, const uint32_t* queue, uint32_t n_queue,
                      uint8_t* prefilter_out, int32_t* node_out, uint8_t* ready_out, bsr_choose_fn choose,
                      bsr_assumed_fn assumed, void* ctx);
void bsr_priority_assumed(void* ctx, const bso_nodes* nd, const bso_pods* pd, uint32_t p, uint32_t n);

/* tests/node_priority_ref.c: its columns, the raw counts, the normalization and the maxima over the fit set */
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

/* the columns of bs_upload_node_locality / bs_upload_pod_locality, the two weights, and scaled[n_images], which
 * bsr_image_spread fills from the node side */
typedef struct {
  const int64_t* image_size;      /* [n_images] */
  const uint32_t* image_bits;     /* [n_images][ceil(n_nodes/32)] */
  const uint64_t* avoid_mask;     /* [n_nodes] */
  uint32_t n_images;
  const uint32_t* image_class;    /* [n_pods] */
  const uint32_t* class_offset;   /* [n_classes + 1] */
  const uint32_t* class_images;   /* [class_offset[n_classes]] */
  const uint8_t* avoid_bit;       /* [n_pods] */
  const int64_t* scaled;          /* [n_images] */
  uint32_t w_img, w_avoid;
} bsr_locality;

static int has_image(const bsr_locality* q, uint32_t n_nodes, uint32_t i, uint32_t n) {
  const uint32_t words = (n_nodes + 31) / 32;
  return (q->image_bits[(size_t)i * words + n / 32] >> (n % 32)) & 1u;
}

/* scaledImageScore: size * (NumNodes / totalNumNodes) in binary64, truncated toward zero by the conversion */
int64_t bsr_image_scaled(int64_t size, uint32_t num_nodes, uint32_t total_nodes) {
  const double spread = (double)num_nodes / (double)total_nodes;
  return (int64_t)((double)size * spread);
}

/* scaled[i] of every name: NumNodes(i) counted node by node over the snapshot */
void bsr_image_spread(const bsr_locality* q, uint32_t n_nodes, int64_t* scaled) {
  for (uint32_t i = 0; i < q->n_images; ++i) {
    uint32_t num = 0;
    for (uint32_t n = 0; n < n_nodes; ++n) num += (uint32_t)has_image(q, n_nodes, i, n);
    scaled[i] = bsr_image_scaled(q->image_size[i], num, n_nodes);
  }
}

/* calculatePriority: the sum clamped to [23 MiB, 1000 MiB], mapped onto 0..100 */
int64_t bsr_image_locality(int64_t sum) {
  const int64_t lo = 23 * BSR_MIB, hi = 1000 * BSR_MIB;
  if (sum < lo) sum = lo;
  else if (sum > hi) sum = hi;
  return 100 * (sum - lo) / (hi - lo);
}

/* IL of pod p on node n: the scaled sizes of the class's ids the node reports, each occurrence counted */
int64_t bsr_il(const bsr_locality* q, const bso_nodes* nd, uint32_t p, uint32_t n) {
  const uint32_t c = q->image_class[p];
  if (c == BSR_IMAGE_NONE) return 0;
  int64_t sum = 0;
  for (uint32_t k = q->class_offset[c]; k < q->class_offset[c + 1]; ++k)
    if (has_image(q, nd->n, q->class_images[k], n)) sum += q->scaled[q->class_images[k]];
  return bsr_image_locality(sum);
}

/* NPA of pod p on node n: 0 when the node's annotation lists the pod's RC / RS controller */
int64_t bsr_npa(const bsr_locality* q, uint32_t p, uint32_t n) {
  const uint8_t b = q->avoid_bit[p];
  if (b == BSR_AVOID_NONE) return 100;
  return ((q->avoid_mask[n] >> b) & 1u) ? 0 : 100;
}

/* the weighted sum of both terms; a column whose weight is 0 is not read (it may be missing) */
uint64_t bsr_locality_term(const bsr_locality* q, const bso_nodes* nd, uint32_t p, uint32_t n) {
  const int64_t il = q->w_img ? bsr_il(q, nd, p, n) : 0;
  const int64_t npa = q->w_avoid ? bsr_npa(q, p, n) : 100;
  return (uint64_t)q->w_img * (uint64_t)il + (uint64_t)q->w_avoid * (uint64_t)npa;
}

/* The list of pod p (as bsr_node_priority_rows): its fitting nodes by the whole score descending, then node index
 * ascending, the first K, padded with node -1 and score INT64_MIN.  s: the ratio setting; pref: the node priorities'
 * columns and weights (NULL: off). */
void bsr_locality_rows(const bsr_locality* q, const bsr_node_pref* pref, const void* s, const bso_nodes* nd,
                       const bso_pods* pd, const int64_t* node_nz, const int64_t* pod_nz, uint32_t p, uint32_t K,
                       uint32_t w_least, uint32_t w_most, uint32_t w_balanced, int32_t* nodes, int64_t* scores) {
  int64_t mt = 0, ma = 0;
  if (pref) bsr_node_pref_maxima(pref, nd, pd, p, &mt, &ma);
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
    sc += bsr_locality_term(q, nd, p, n);
    const int64_t v = (int64_t)sc;
    uint32_t pos = 0;
    while (pos < filled && scores[pos] >= v) ++pos;
    if (pos >= K) continue;
    for (uint32_t k = (filled < K ? filled : K - 1); k > pos; --k) { nodes[k] = nodes[k - 1]; scores[k] = scores[k - 1]; }
    nodes[pos] = (int32_t)n;
    scores[pos] = v;
    if (filled < K) ++filled;
  }
}

/* The chooser for bsr_replay_choose: the live non-zero column (first member, so that tests/replay_priority_ref.c's
 * bsr_priority_assumed grows it on every assume), the ratio setting and the locality columns */
typedef struct {
  int64_t* node_nz;
  const int64_t* pod_nz;
  uint32_t w_least, w_most, w_balanced;
  const void* s;
  const bsr_locality* q;
} bsr_locality_ctx;

int32_t bsr_locality_choose(void* ctx, const bso_nodes* nd, const bso_pods* pd, uint32_t p) {
  const bsr_locality_ctx* c = (const bsr_locality_ctx*)ctx;
  int32_t best = -1;
  int64_t best_s = INT64_MIN;
  for (uint32_t n = 0; n < nd->n; ++n) {
    if (!bso_fit_eval(nd, pd, p, n, NULL)) continue;
    const int64_t sc = (int64_t)((uint64_t)bsr_ratio_total(c->s, nd, pd, c->node_nz, c->pod_nz, p, n, c->w_least,
                                                           c->w_most, c->w_balanced) +
                                 bsr_locality_term(c->q, nd, p, n));
    if (best < 0 || sc > best_s) { best = (int32_t)n; best_s = sc; }   /* ascending nodes: ties keep the lower index */
  }
  return best;
}

/* bs_replay_priority with the locality terms: node_nz [2][n_nodes] is the live column, updated in place */
int bsr_replay_locality(bso_nodes* nd, const bso_pods* pd, bso_groups* gr, const uint32_t* queue, uint32_t n_queue,
                        uint8_t* prefilter_out, int32_t* node_out, uint8_t* ready_out, int64_t* node_nz,
                        const int64_t* pod_nz, uint32_t w_least, uint32_t w_most, uint32_t w_balanced, const void* s,
                        const bsr_locality* q) {
  bsr_locality_ctx c = {node_nz, pod_nz, w_least, w_most, w_balanced, s, q};
  return bsr_replay_choose(nd, pd, gr, queue, n_queue, prefilter_out, node_out, ready_out, bsr_locality_choose,
                           bsr_priority_assumed, &c);
}
