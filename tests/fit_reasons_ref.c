/* fit_reasons_ref.c — TEST INFRASTRUCTURE: the CPU restatement of the reason rows (include/bsched.h BS_OUT_REASONS),
 * built on the oracle's line-by-line helpers (oracle/bs_oracle.h: bso_check_fit, bso_single_node_resource,
 * bso_pod_require) and linked against oracle/libbs_oracle.so.  tests/native.py compiles it with the other
 * restatements and tests/fit_reasons_ref.py binds it. */
#include <stdint.h>
#include <string.h>

#include "bs_oracle.h"

/* core.go:606-617: nil info, nil Node(), Spec.Unschedulable */
static int node_skipped(const bso_nodes* nd, uint32_t i) {
  return (nd->flags[i] & (BSO_NODE_NIL | BSO_NODE_NO_NODE | BSO_NODE_UNSCHEDULABLE)) != 0;
}

/* Reason row of pod p: counts[4 + lanes], one bin per reason, over every node.  Guards in the reference's order
 * (nil, Node() == nil, unschedulable: core.go:606-617; the Taints() error, :639), each guarded node in one bin; past
 * the guards checkFit's two predicates each add their reason (:741-759); past checkFit every lane of
 * compareResourceAndRequire (:672-699) that is short adds its reason, with `left` = singleNodeResource at percent 1.0
 * and the request of getPodResourceRequire. */
void bsr_fit_reasons(const bso_nodes* nd, const bso_pods* pd, uint32_t p, uint32_t* counts) {
  const uint32_t L = nd->lanes;
  const uint64_t sel = pd->sel_mask[p], tol = pd->tol_mask[p];
  const uint32_t aff = pd->aff_class ? pd->aff_class[p] : BSO_AFF_NONE;
  memset(counts, 0, sizeof(uint32_t) * (4 + L));
  bso_resource req, left;
  bso_pod_require(pd, p, &req);
  for (uint32_t n = 0; n < nd->n; ++n) {
    const uint8_t f = nd->flags[n];
    if (node_skipped(nd, n)) {
      if (f & (BSO_NODE_NIL | BSO_NODE_NO_NODE)) counts[1]++;
      else counts[0]++;
      continue;
    }
    if (f & BSO_NODE_TAINTS_ERR) { counts[1]++; continue; }
    /* bso_check_fit's two predicates, each giving its own reason: PodMatchNodeSelector (label bits and the
     * affinity-class bit; tolerating the node's own taints leaves only the selector) and PodToleratesNodeTaints */
    const int sel_ok = bso_check_fit(nd, n, sel, nd->taint_mask[n], aff);
    const int taint_ok = (nd->taint_mask[n] & ~tol) == 0;
    if (!sel_ok) counts[2]++;
    if (!taint_ok) counts[3]++;
    if (!sel_ok || !taint_ok) continue;
    bso_single_node_resource(nd, n, sel, tol, aff, 1.0f, &left);
    for (uint32_t d = 0; d < L; ++d) {
      int shrt;
      if (d < 4) shrt = left.v[d] < req.v[d];
      else {
        const uint32_t bit = 1u << d;
        if (!(req.present & bit)) continue;                                 /* :686 keys of req only */
        shrt = (left.present & bit) ? req.v[d] > left.v[d] : req.v[d] != 0;   /* :694 / :688-692 */
      }
      if (shrt) counts[4 + d]++;
    }
  }
}
