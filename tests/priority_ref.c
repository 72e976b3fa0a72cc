/* priority_ref.c — TEST INFRASTRUCTURE: the CPU restatement of the priority lists (include/bsched.h BS_OUT_PRIORITY).
 * The fit set comes from the oracle's bso_fit_eval (oracle/bs_oracle.h); the three scorers restate kube-scheduler
 * v1.17's NodeResourcesLeastAllocated, NodeResourcesMostAllocated and NodeResourcesBalancedAllocation [upstream, from
 * memory].  Compiled with -ffp-contract=off, so every double operation rounds on its own.  tests/native.py compiles
 * it with the other restatements and tests/priority_ref.py binds it. */
#include <math.h>
#include <stddef.h>
#include <stdint.h>

#include "bs_oracle.h"
#include "bs_ref.h"

/* leastRequestedScore / mostRequestedScore: int64, truncating */
static int64_t least_score(int64_t r, int64_t c) {
  if (c == 0 || r > c) return 0;
  return ((c - r) * 100) / c;
}
static int64_t most_score(int64_t r, int64_t c) {
  if (c == 0 || r > c) return 0;
  return (r * 100) / c;
}
/* fractionOfCapacity */
static double fraction(int64_t r, int64_t c) { return c == 0 ? 1.0 : (double)r / (double)c; }
/* int64(x) toward zero; the products reach below -2^63 only with a negative allocatable, and saturate there */
static int64_t to_int64(double x) { return x < -9223372036854775808.0 ? INT64_MIN : (int64_t)x; }

int64_t bsr_priority_score(int64_t r_cpu, int64_t c_cpu, int64_t r_mem, int64_t c_mem, uint32_t w_least, uint32_t w_most,
                           uint32_t w_balanced) {
  const int64_t least = (least_score(r_cpu, c_cpu) + least_score(r_mem, c_mem)) / 2;
  const int64_t most = (most_score(r_cpu, c_cpu) + most_score(r_mem, c_mem)) / 2;
  const double fc = fraction(r_cpu, c_cpu), fm = fraction(r_mem, c_mem);
  int64_t balanced = 0;
  if (!(fc >= 1 || fm >= 1)) {
    const double diff = fabs(fc - fm);
    balanced = to_int64((1 - diff) * 100.0);
  }
  /* int64 sums wrap as Go's do */
  const uint64_t s = (uint64_t)w_least * (uint64_t)least + (uint64_t)w_most * (uint64_t)most +
                     (uint64_t)w_balanced * (uint64_t)balanced;
  return (int64_t)s;
}

/* The list of pod p: its fitting nodes (bso_fit_eval) by score descending, then node index ascending, the first K of
 * them, padded with node -1 and score INT64_MIN.  node_nz [2][n_nodes], pod_nz [2][n_pods]: cpu, memory. */
void bsr_priority_rows(const bso_nodes* nd, const bso_pods* pd, const int64_t* node_nz, const int64_t* pod_nz, uint32_t p,
                       uint32_t K, uint32_t w_least, uint32_t w_most, uint32_t w_balanced, int32_t* nodes, int64_t* scores) {
  uint32_t filled = 0;
  for (uint32_t k = 0; k < K; ++k) { nodes[k] = -1; scores[k] = INT64_MIN; }
  for (uint32_t n = 0; n < nd->n; ++n) {
    int64_t unused;
    if (!bso_fit_eval(nd, pd, p, n, &unused)) continue;
    const int64_t r_cpu = node_nz[n] + pod_nz[p], r_mem = node_nz[nd->n + n] + pod_nz[pd->n + p];
    const int64_t s = bsr_priority_score(r_cpu, nd->alloc[n], r_mem, nd->alloc[(size_t)nd->n + n], w_least, w_most,
                                         w_balanced);
    /* nodes arrive in ascending order: a node goes after every entry of equal or higher score */
    uint32_t pos = 0;
    while (pos < filled && scores[pos] >= s) ++pos;
    if (pos >= K) continue;
    for (uint32_t k = (filled < K ? filled : K - 1); k > pos; --k) { nodes[k] = nodes[k - 1]; scores[k] = scores[k - 1]; }
    nodes[pos] = (int32_t)n;
    scores[pos] = s;
    if (filled < K) ++filled;
  }
}
