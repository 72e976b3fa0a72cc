/* replay_priority_ref.c — TEST INFRASTRUCTURE: the CPU restatement of bs_replay_priority (include/bsched.h).
 *
 * bsr_replay_choose is the oracle's pod-at-a-time walk (oracle/bs_oracle.c bso_replay) built from the oracle's public
 * line-by-line helpers, with the node choice as a hook: the chooser returns a node where bso_fit_eval holds on the live
 * tables, or -1, and is told which node the pod was assumed onto.  With bsr_first_fit it is bso_replay, which the
 * tests check; with bsr_priority_choose it is bs_replay_priority: among the fitting nodes the highest
 * bsr_priority_score (tests/priority_ref.c) over a live copy of the node non-zero column, ties to the lower index.
 * tests/replay_priority_ref.py compiles it with priority_ref.c into a temporary directory and binds it. */
#include <stddef.h>
#include <stdint.h>

#include "bs_oracle.h"

#define LANE_PODS 3
#define POD_AFF(pd, p) ((pd)->aff_class ? (pd)->aff_class[p] : BSO_AFF_NONE)
#define GROUP_AFF(gr, g) ((gr)->rep_aff ? (gr)->rep_aff[g] : BSO_AFF_NONE)

int64_t bsr_priority_score(int64_t r_cpu, int64_t c_cpu, int64_t r_mem, int64_t c_mem, uint32_t w_least, uint32_t w_most,
                           uint32_t w_balanced);

typedef int32_t (*bsr_choose_fn)(void* ctx, const bso_nodes* nd, const bso_pods* pd, uint32_t p);
typedef void (*bsr_assumed_fn)(void* ctx, const bso_nodes* nd, const bso_pods* pd, uint32_t p, uint32_t n);

/* bso_replay's node choice: the first node in list order where the pod fits */
int32_t bsr_first_fit(void* ctx, const bso_nodes* nd, const bso_pods* pd, uint32_t p) {
  (void)ctx;
  for (uint32_t n = 0; n < nd->n; ++n)
    if (bso_fit_eval(nd, pd, p, n, NULL)) return (int32_t)n;
  return -1;
}

/* The scoring chooser's state: node_nz [2][n_nodes] is the LIVE column (grown on every assume), pod_nz [2][n_pods]. */
typedef struct {
  int64_t* node_nz;
  const int64_t* pod_nz;
  uint32_t w_least, w_most, w_balanced;
} bsr_priority_ctx;

int32_t bsr_priority_choose(void* ctx, const bso_nodes* nd, const bso_pods* pd, uint32_t p) {
  const bsr_priority_ctx* c = (const bsr_priority_ctx*)ctx;
  int32_t best = -1;
  int64_t best_s = INT64_MIN;
  for (uint32_t n = 0; n < nd->n; ++n) {
    if (!bso_fit_eval(nd, pd, p, n, NULL)) continue;
    const int64_t s = bsr_priority_score(c->node_nz[n] + c->pod_nz[p], nd->alloc[n],
                                         c->node_nz[(size_t)nd->n + n] + c->pod_nz[(size_t)pd->n + p],
                                         nd->alloc[(size_t)nd->n + n], c->w_least, c->w_most, c->w_balanced);
    if (best < 0 || s > best_s) { best = (int32_t)n; best_s = s; }   /* ascending nodes: ties keep the lower index */
  }
  return best;
}

/* NodeInfo.AddPod grows the node's non-zero requests by the pod's */
void bsr_priority_assumed(void* ctx, const bso_nodes* nd, const bso_pods* pd, uint32_t p, uint32_t n) {
  bsr_priority_ctx* c = (bsr_priority_ctx*)ctx;
  c->node_nz[n] += c->pod_nz[p];
  c->node_nz[(size_t)nd->n + n] += c->pod_nz[(size_t)pd->n + p];
}

/* bso_replay with the node choice `choose` (assumed may be NULL); tables mutated in place as bso_replay does */
int bsr_replay_choose(bso_nodes* nd, const bso_pods* pd, bso_groups* gr, const uint32_t* queue, uint32_t n_queue,
                      uint8_t* prefilter_out, int32_t* node_out, uint8_t* ready_out, bsr_choose_fn choose,
                      bsr_assumed_fn assumed, void* ctx) {
  const uint32_t N = nd->n, L = nd->lanes;
  for (uint32_t qi = 0; qi < n_queue; ++qi) {
    const uint32_t p = queue[qi];
    const int g = pd->gid[p];
    node_out[qi] = -1;
    ready_out[qi] = 0;
    /* ---- PreFilter, core.go:88-167, against live state ---- */
    uint8_t code = BSO_PF_PASS;
    do {
      if (g == BSO_GID_NONE) break;
      if (pd->flags[p] & BSO_POD_PERMITTED_RECENTLY) break;
      if (g < 0 || (uint32_t)g >= gr->n) { code = BSO_PF_NOT_FOUND; break; }
      if (gr->flags[g] & BSO_GROUP_DENIED) { code = BSO_PF_DENIED; break; }
      /* fillOccupiedObj :486-493 */
      if (!(gr->flags[g] & BSO_GROUP_HAS_POD)) {
        gr->flags[g] |= BSO_GROUP_HAS_POD;
        gr->rep_sel[g] = pd->sel_mask[p];
        gr->rep_tol[g] = pd->tol_mask[p];
        if (gr->rep_aff) gr->rep_aff[g] = POD_AFF(pd, p);
      }
      if (!(gr->flags[g] & BSO_GROUP_HAS_MINRES)) {
        gr->flags[g] |= BSO_GROUP_HAS_MINRES;
        for (uint32_t d = 0; d < L; ++d) {
          const int pres = d < 4 || (pd->req_present[p] & (1u << d));
          gr->min_res[(size_t)d * gr->n + g] = pres ? pd->req[(size_t)d * pd->n + p] : 0;
        }
        gr->min_res_present[g] = pd->req_present[p] & ~0xFu;
      }
      if (pd->flags[p] & BSO_POD_OCC_NOREFS) { code = BSO_PF_OCC_NOREFS; break; }
      if (pd->flags[p] & BSO_POD_OCC_MISMATCH) { code = BSO_PF_OCCUPIED; break; }
      uint32_t mf;
      int pn;
      const int m = bso_find_max_pg(gr, &mf, &pn);
      if (m < 0) break;
      const uint32_t matched = gr->matched[m];
      bso_resource need, req;
      if (matched == 0) {
        bso_pre_allocated(gr, (uint32_t)g, 0, &need);
        if (!bso_compare_cluster(nd, gr->rep_sel[g], gr->rep_tol[g], GROUP_AFF(gr, g), &need, 1.0f)) {
          gr->flags[g] |= BSO_GROUP_DENIED;
          code = BSO_PF_NOT_ENOUGH;
        }
        break;
      }
      if (m == g) break;
      bso_pre_allocated(gr, (uint32_t)m, (int64_t)matched, &need);
      bso_pod_require(pd, p, &req);
      bso_resource_add(&need, &req, L);
      if (!bso_compare_cluster(nd, gr->rep_sel[m], gr->rep_tol[m], GROUP_AFF(gr, m), &need, 0.7f)) {
        gr->flags[g] |= BSO_GROUP_DENIED;
        code = BSO_PF_NOT_ENOUGH;
      }
    } while (0);
    prefilter_out[qi] = code;
    if (code != BSO_PF_PASS) continue;
    const int32_t chosen = choose(ctx, nd, pd, p);
    node_out[qi] = chosen;
    if (chosen < 0) continue;
    /* assume: NodeInfo.AddPod adds the pod's resources to requested */
    for (uint32_t d = 0; d < L; ++d) {
      if (d == LANE_PODS) continue;
      if (d >= 4 && !(pd->req_present[p] & (1u << d))) continue;
      nd->requested[(size_t)d * N + chosen] += pd->req[(size_t)d * pd->n + p];
      if (d >= 4) nd->req_present[chosen] |= 1u << d;
    }
    nd->pod_count[chosen] += 1;
    if (assumed) assumed(ctx, nd, pd, p, (uint32_t)chosen);
    /* ---- Permit, core.go:268-309 ---- */
    if (g < 0 || (uint32_t)g >= gr->n) { ready_out[qi] = 1; continue; }
    gr->matched[g] += 1; /* :290 MatchedPodNodes.Set */
    if (bso_permit_ready(gr->matched[g], gr->min_member[g], gr->scheduled[g])) {
      gr->flags[g] |= BSO_GROUP_SCHEDULED; /* :305 */
      ready_out[qi] = 1;
    }
  }
  return 0;
}

/* bs_replay_priority: node_nz [2][n_nodes] is the live column, updated in place */
int bsr_replay_priority(bso_nodes* nd, const bso_pods* pd, bso_groups* gr, const uint32_t* queue, uint32_t n_queue,
                        uint8_t* prefilter_out, int32_t* node_out, uint8_t* ready_out, int64_t* node_nz,
                        const int64_t* pod_nz, uint32_t w_least, uint32_t w_most, uint32_t w_balanced) {
  bsr_priority_ctx c = {node_nz, pod_nz, w_least, w_most, w_balanced};
  return bsr_replay_choose(nd, pd, gr, queue, n_queue, prefilter_out, node_out, ready_out, bsr_priority_choose,
                           bsr_priority_assumed, &c);
}
