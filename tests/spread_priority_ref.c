/* spread_priority_ref.c — TEST INFRASTRUCTURE: the CPU restatement of kube-scheduler v1.17's SelectorSpread priority
 * as the engine adds it to the priority lists (include/bsched.h bs_set_spread_weight), written from
 * selector_spreading.go's CalculateSpreadPriorityMap and CalculateSpreadPriorityReduce [upstream, from memory].  The
 * reduce runs over the pod's fit set as upstream runs over the filtered nodes: the largest count, a map from zone to
 * summed count that every zoned node of the set enters (count 0 included), and haveZones = the map is not empty.  The
 * rest of the score is tests/ratio_priority_ref.c's bsr_ratio_total plus, when given, the TaintToleration and
 * NodeAffinity terms of tests/node_priority_ref.c and the locality terms of tests/locality_priority_ref.c, so every
 * flag combination of the lists has a restatement.  tests/spread_priority_ref.py compiles it with -ffp-contract=off
 * into a library of its own, linked against those libraries and the oracle. */
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>

#include "bs_oracle.h"

#define BSR_SPREAD_NONE 0xffffffffu
#define BSR_ZONE_NONE 0xffu
#define BSR_ZONES 256

/* tests/ratio_priority_ref.c (tests/native.py's library) */
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

/* tests/locality_priority_ref.c: its columns stay opaque here (scaled[] filled by the caller) */
uint64_t bsr_locality_term(const void* q, const bso_nodes* nd, uint32_t p, uint32_t n);

/* the columns of bs_upload_node_spread / bs_upload_pod_spread and the weight */
typedef struct {
  const uint8_t* zone;            /* [n_nodes] */
  const int32_t* counts;          /* [n_classes][n_nodes] */
  const uint32_t* spread_class;   /* [n_pods] */
  uint32_t w_spread;
} bsr_spread;

/* CalculateSpreadPriorityMap: the matching pods on the node; 0 for a pod without selectors */
int64_t bsr_spread_count(const bsr_spread* q, uint32_t n_nodes, uint32_t p, uint32_t n) {
  const uint32_t c = q->spread_class[p];
  return c == BSR_SPREAD_NONE ? 0 : q->counts[(size_t)c * n_nodes + n];
}

/* the score of one node: fScore from the node's count, blended with the zone's score when the node is zoned and
 * haveZones; every operation a binary64 rounding of its own (-ffp-contract=off), then truncation toward zero */
int64_t bsr_spread_score(int64_t max_node, int64_t count, int zoned, int64_t max_zone, int64_t zone_count) {
  const double zone_weighting = 2.0 / 3.0;
  double f = 100.0;
  if (max_node > 0) f = 100.0 * ((double)(max_node - count) / (double)max_node);
  if (zoned) {
    double zs = 100.0;
    if (max_zone > 0) zs = 100.0 * ((double)(max_zone - zone_count) / (double)max_zone);
    f = (f * (1.0 - zone_weighting)) + (zone_weighting * zs);
  }
  return (int64_t)f;
}

/* CalculateSpreadPriorityReduce over the fit set of pod p: ss[n] for every fitting node n (others untouched) */
void bsr_spread_reduce(const bsr_spread* q, const bso_nodes* nd, const bso_pods* pd, uint32_t p, int64_t* ss) {
  int64_t by_zone[BSR_ZONES] = {0};
  uint8_t in_map[BSR_ZONES] = {0};
  int64_t max_node = 0;
  for (uint32_t n = 0; n < nd->n; ++n) {
    if (!bso_fit_eval(nd, pd, p, n, NULL)) continue;
    const int64_t c = bsr_spread_count(q, nd->n, p, n);
    if (c > max_node) max_node = c;
    const uint8_t z = q->zone[n];
    if (z == BSR_ZONE_NONE) continue;
    by_zone[z] += c;   /* countsByZone[zoneID] += count: the entry exists even for count 0 */
    in_map[z] = 1;
  }
  int have_zones = 0;
  int64_t max_zone = 0;
  for (int z = 0; z < BSR_ZONES; ++z)
    if (in_map[z]) {
      have_zones = 1;
      if (by_zone[z] > max_zone) max_zone = by_zone[z];
    }
  for (uint32_t n = 0; n < nd->n; ++n) {
    if (!bso_fit_eval(nd, pd, p, n, NULL)) continue;
    const uint8_t z = q->zone[n];
    const int zoned = have_zones && z != BSR_ZONE_NONE;
    ss[n] = bsr_spread_score(max_node, bsr_spread_count(q, nd->n, p, n), zoned, max_zone, zoned ? by_zone[z] : 0);
  }
}

/* The list of pod p (as bsr_locality_rows): its fitting nodes by the whole score descending, then node index
 * ascending, the first K, padded with node -1 and score INT64_MIN.  s: the ratio setting; pref: the node priorities'
 * columns and weights; loc: the locality columns and weights (NULL: off, either). */
void bsr_spread_rows(const bsr_spread* q, const bsr_node_pref* pref, const void* loc, const void* s,
                     const bso_nodes* nd, const bso_pods* pd, const int64_t* node_nz, const int64_t* pod_nz,
                     uint32_t p, uint32_t K, uint32_t w_least, uint32_t w_most, uint32_t w_balanced, int32_t* nodes,
                     int64_t* scores) {
  int64_t mt = 0, ma = 0;
  if (pref) bsr_node_pref_maxima(pref, nd, pd, p, &mt, &ma);
  int64_t* ss = (int64_t*)calloc(nd->n ? nd->n : 1, sizeof(int64_t));
  if (q->w_spread) bsr_spread_reduce(q, nd, pd, p, ss);
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
    sc += (uint64_t)q->w_spread * (uint64_t)ss[n];
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
}
