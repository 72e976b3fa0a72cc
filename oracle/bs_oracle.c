/*
 * bs_oracle.c — TEST INFRASTRUCTURE, NOT PRODUCT (see bs_oracle.h).
 *
 * Plain-C restatement of pkg/scheduler/core/core.go of tenstack/batch-scheduler.
 * Each function cites the lines it follows.  Integer widths follow Go on amd64:
 * int == int64, uint32 arithmetic wraps, float32 multiply is a single RN
 * multiply, float32 -> int64 conversion truncates.
 *
 * build: see oracle/Makefile (gcc -O2 -ffp-contract=off -fopenmp).
 */
#include "bs_oracle.h"

#include <limits.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#define LANE_CPU 0
#define LANE_MEM 1
#define LANE_EPH 2
#define LANE_PODS 3

#define POD_AFF(pd, p) ((pd)->aff_class ? (pd)->aff_class[p] : BSO_AFF_NONE)
#define GROUP_AFF(gr, g) ((gr)->rep_aff ? (gr)->rep_aff[g] : BSO_AFF_NONE)

static inline int64_t wrap_add(int64_t a, int64_t b) { return (int64_t)((uint64_t)a + (uint64_t)b); }
static inline int64_t wrap_sub(int64_t a, int64_t b) { return (int64_t)((uint64_t)a - (uint64_t)b); }
static inline int64_t wrap_mul(int64_t a, int64_t b) { return (int64_t)((uint64_t)a * (uint64_t)b); }

int bso_max_threads(void) {
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}

/* core.go:656-659,667 — int64(float32(alloc) * percent).  volatile keeps the
 * product a true float32 (no excess precision, no contraction). */
int64_t bso_scale(int64_t alloc, float percent) {
  volatile float f = (float)alloc;
  volatile float prod = f * percent;
  return (int64_t)prod;
}

/* core.go:741-759 checkFit: PodMatchNodeSelector && PodToleratesNodeTaints, with
 * both predicates pre-encoded by the packer: every required label bit is on the
 * node, and every NoSchedule/NoExecute taint bit of the node is tolerated. */
int bso_check_fit(const bso_nodes* nd, uint32_t i, uint64_t sel, uint64_t tol, uint32_t aff) {
  if ((nd->label_mask[i] & sel) != sel) return 0;
  if ((nd->taint_mask[i] & ~tol) != 0) return 0;
  /* the part of PodMatchNodeSelector bit masks cannot carry (required nodeAffinity terms): one
   * host-evaluated bit per (affinity class, node), see include/bsched.h bs_upload_affinity */
  if (aff != BSO_AFF_NONE) {
    if (!nd->aff_bits || aff >= nd->n_aff) return 0;
    const uint32_t W = (nd->n + 31) / 32;
    if (!((nd->aff_bits[(size_t)aff * W + (i >> 5)] >> (i & 31)) & 1u)) return 0;
  }
  return 1;
}

/* core.go:634-670 singleNodeResource */
void bso_single_node_resource(const bso_nodes* nd, uint32_t i, uint64_t sel, uint64_t tol, uint32_t aff,
                              float percent, bso_resource* out) {
  const uint32_t n = nd->n, L = nd->lanes;
  memset(out, 0, sizeof(*out)); /* :635-637 empty resource, empty scalar map */
  if (nd->flags[i] & BSO_NODE_TAINTS_ERR) return; /* :639-641 */
  if (!bso_check_fit(nd, i, sel, tol, aff)) return; /* :642-645 */
  /* :650-653 podCount = requested.AllowedPodNumber, or len(info.Pods()) when 0 */
  int64_t pod_count = nd->requested[(size_t)LANE_PODS * n + i];
  if (pod_count == 0) pod_count = nd->pod_count[i];
  /* :656-659 */
  out->v[LANE_PODS] = wrap_sub(bso_scale(nd->alloc[(size_t)LANE_PODS * n + i], percent), pod_count);
  out->v[LANE_CPU] = wrap_sub(bso_scale(nd->alloc[(size_t)LANE_CPU * n + i], percent),
                              nd->requested[(size_t)LANE_CPU * n + i]);
  out->v[LANE_MEM] = wrap_sub(bso_scale(nd->alloc[(size_t)LANE_MEM * n + i], percent),
                              nd->requested[(size_t)LANE_MEM * n + i]);
  out->v[LANE_EPH] = wrap_sub(bso_scale(nd->alloc[(size_t)LANE_EPH * n + i], percent),
                              nd->requested[(size_t)LANE_EPH * n + i]);
  /* :662-668 scalar keys of allocatable that also exist in requested */
  for (uint32_t d = 4; d < L; ++d) {
    const uint32_t bit = 1u << d;
    if (!(nd->alloc_present[i] & bit)) continue;
    if (!(nd->req_present[i] & bit)) continue; /* :663-666 */
    out->v[d] = wrap_sub(bso_scale(nd->alloc[(size_t)d * n + i], percent),
                         nd->requested[(size_t)d * n + i]);
    out->present |= bit;
  }
}

/* core.go:672-699 compareResourceAndRequire */
int bso_compare_resource_and_require(const bso_resource* left, const bso_resource* req,
                                     uint32_t lanes) {
  if (left->v[LANE_MEM] < req->v[LANE_MEM]) return 0;   /* :673 */
  if (left->v[LANE_CPU] < req->v[LANE_CPU]) return 0;   /* :676 */
  if (left->v[LANE_EPH] < req->v[LANE_EPH]) return 0;   /* :679 */
  if (left->v[LANE_PODS] < req->v[LANE_PODS]) return 0; /* :683 */
  for (uint32_t d = 4; d < lanes; ++d) {                /* :686 keys of req only */
    const uint32_t bit = 1u << d;
    if (!(req->present & bit)) continue;
    if (!(left->present & bit)) {                       /* :688-692 */
      if (req->v[d] != 0) return 0;
      continue;
    }
    if (req->v[d] > left->v[d]) return 0;               /* :694 */
  }
  return 1;
}

/* nodeinfo.Resource.Add(x.ResourceList()) — k8s v1.17.5 [restated]: the four
 * fixed fields always appear in ResourceList and add exactly; every scalar key
 * of x is added and becomes present in the accumulator (AddScalar/SetScalar). */
void bso_resource_add(bso_resource* acc, const bso_resource* x, uint32_t lanes) {
  for (uint32_t d = 0; d < 4; ++d) acc->v[d] = wrap_add(acc->v[d], x->v[d]);
  for (uint32_t d = 4; d < lanes; ++d) {
    const uint32_t bit = 1u << d;
    if (!(x->present & bit)) continue;
    acc->v[d] = wrap_add(acc->v[d], x->v[d]);
    acc->present |= bit;
  }
}

static inline int node_skipped(const bso_nodes* nd, uint32_t i) {
  /* core.go:606-617: nil info, nil Node(), Spec.Unschedulable */
  return (nd->flags[i] & (BSO_NODE_NIL | BSO_NODE_NO_NODE | BSO_NODE_UNSCHEDULABLE)) != 0;
}

/* core.go:595-632 compareClusterResourceAndRequire */
int bso_compare_cluster(const bso_nodes* nd, uint64_t sel, uint64_t tol, uint32_t aff, const bso_resource* need,
                        float percent) {
  bso_resource running, left;
  memset(&running, 0, sizeof(running)); /* :602 */
  for (uint32_t i = 0; i < nd->n; ++i) { /* :604 snapshot list order */
    if (node_skipped(nd, i)) continue;   /* :606-617 */
    bso_single_node_resource(nd, i, sel, tol, aff, percent, &left); /* :619 */
    bso_resource_add(&running, &left, nd->lanes);              /* :621 */
    if (bso_compare_resource_and_require(&running, need, nd->lanes)) return 1; /* :623-627 */
  }
  return 0; /* :631 */
}

/* core.go:566-593 computeClusterResource (no early exit; log argument only) */
void bso_compute_cluster(const bso_nodes* nd, uint64_t sel, uint64_t tol, uint32_t aff, bso_resource* out) {
  bso_resource left;
  memset(out, 0, sizeof(*out));
  for (uint32_t i = 0; i < nd->n; ++i) {
    if (node_skipped(nd, i)) continue;
    bso_single_node_resource(nd, i, sel, tol, aff, 1.0f, &left);
    bso_resource_add(out, &left, nd->lanes);
  }
}

/* core.go:701-739 findMaxPG, iterating in table-index order (the reference
 * ranges over a Go map, so its tie order is random: quirk Q8). */
static int find_max_pg_flags(const bso_groups* gr, const uint8_t* flags, uint32_t* max_finished,
                             int* panic) {
  int max_idx = -1;
  uint32_t max_fin = 0;
  if (panic) *panic = 0;
  for (uint32_t g = 0; g < gr->n; ++g) {
    uint32_t finished = 0;
    if (flags[g] & BSO_GROUP_SCHEDULED) continue;   /* :706 */
    if (!(flags[g] & BSO_GROUP_HAS_POD)) continue;  /* :709 */
    const uint32_t mm = gr->min_member[g], sc = gr->scheduled[g];
    if ((uint32_t)(mm - sc) <= 0u) {                /* :712-714 uint32: true only when equal */
      finished = 0;
    } else {
      if (mm == 0) {                                /* :716-717 integer divide by zero */
        if (panic) *panic = 1;
        continue;
      }
      finished = (uint32_t)((uint32_t)(gr->matched[g] + sc) * 1000u) / mm; /* :716-717 */
    }
    if (finished > max_fin) {                       /* :721 */
      max_fin = finished;
      max_idx = (int)g;
    } else if (finished == max_fin) {               /* :725 */
      if (max_idx < 0 ||
          (gr->scheduled[max_idx] >= gr->min_member[max_idx] && sc == 0)) { /* :729-731 */
        max_fin = finished;
        max_idx = (int)g;
      }
    }
  }
  if (max_finished) *max_finished = max_fin;
  return max_idx;
}

int bso_find_max_pg(const bso_groups* gr, uint32_t* max_finished, int* panic) {
  return find_max_pg_flags(gr, gr->flags, max_finished, panic);
}

/* core.go:774-793 getPreAllocatedResource, over explicit MinResources columns */
static void pre_allocated_cols(const bso_groups* gr, uint32_t g, int64_t matched, int has_minres,
                               const int64_t* min_res, uint32_t min_res_present,
                               bso_resource* out) {
  memset(out, 0, sizeof(*out));
  int64_t not_finished;
  if (matched != 0) not_finished = (int64_t)gr->min_member[g] - matched;        /* :778-779 */
  else not_finished = (int64_t)gr->min_member[g] - (int64_t)gr->scheduled[g];   /* :780-783 */
  if (not_finished > 0 && has_minres) { /* :784-788: notFinished x Add(MinResources) */
    for (uint32_t d = 0; d < gr->lanes; ++d) {
      if (d >= 4 && !(min_res_present & (1u << d))) continue;
      out->v[d] = wrap_mul(min_res[d], not_finished);
    }
    out->present = min_res_present;
  }
  if (out->v[LANE_PODS] == 0) out->v[LANE_PODS] = (int64_t)gr->min_member[g] + 1; /* :789-791 */
}

void bso_pre_allocated(const bso_groups* gr, uint32_t g, int64_t matched, bso_resource* out) {
  int64_t mr[BSO_MAX_LANES];
  for (uint32_t d = 0; d < gr->lanes; ++d) mr[d] = gr->min_res[(size_t)d * gr->n + g];
  pre_allocated_cols(gr, g, matched, (gr->flags[g] & BSO_GROUP_HAS_MINRES) != 0, mr,
                     gr->min_res_present[g], out);
}

/* core.go:761-772 getPodResourceRequire — the container sum is done by the
 * packer; the table row is the resulting nodeinfo.Resource. */
void bso_pod_require(const bso_pods* pd, uint32_t p, bso_resource* out) {
  memset(out, 0, sizeof(*out));
  for (uint32_t d = 0; d < pd->lanes; ++d) {
    if (d >= 4 && !(pd->req_present[p] & (1u << d))) continue;
    out->v[d] = pd->req[(size_t)d * pd->n + p];
  }
  out->present = pd->req_present[p] & ~0xFu;
}

/* core.go:303 ready := uint32(len(Items())) >= MinMember - Status.Scheduled */
int bso_permit_ready(uint32_t matched_count, uint32_t min_member, uint32_t scheduled) {
  return matched_count >= (uint32_t)(min_member - scheduled);
}

/* core.go:368-411 Compare */
int bso_compare(const bso_pods* pd, const bso_groups* gr, uint32_t a, uint32_t b) {
  const int32_t prio1 = pd->priority[a], prio2 = pd->priority[b];
  const int g1 = pd->gid[a], g2 = pd->gid[b];
  const int name1_empty = (g1 == BSO_GID_NONE), name2_empty = (g2 == BSO_GID_NONE);
  if (prio1 > prio2) return 1;                                   /* :379 */
  if (prio1 == prio2) {                                          /* :383 */
    if (name1_empty && name2_empty) return pd->ts_ns[a] < pd->ts_ns[b]; /* :384-386 */
    if (name1_empty) return 1;                                   /* :388 */
    if (name2_empty) return 0;                                   /* :391 */
  }
  /* :395-399 lister lookups; Get("") or an unknown group is an error */
  /* a group index outside the table is an unknown group as well */
  const int miss1 = name1_empty || g1 < 0 || (uint32_t)g1 >= gr->n || (pd->flags[a] & BSO_POD_LISTER_MISS);
  const int miss2 = name2_empty || g2 < 0 || (uint32_t)g2 >= gr->n || (pd->flags[b] & BSO_POD_LISTER_MISS);
  if (miss1 || miss2) return 0;
  const int64_t c1 = gr->creation_ns[g1], c2 = gr->creation_ns[g2];
  const uint32_t r1 = gr->name_rank[g1], r2 = gr->name_rank[g2];
  if (prio1 == prio2 && c1 < c2) return 1;                       /* :400 */
  if (prio1 == prio2 && c1 == c2 && r1 > r2) return 1;           /* :404 pgName1 > pgName2 */
  return prio1 == prio2 && c1 == c2 && r1 == r2 && pd->ts_ns[a] < pd->ts_ns[b]; /* :407 */
}

/* Total order used for the round's `order` output: identical to Compare on
 * well-formed pods; pods whose lister lookup fails (Compare answers false both
 * ways, which is not a strict weak order) sort after every resolvable grouped
 * pod of the same priority, by timestamp.  Ties keep table order. */
static int key_less(const bso_pods* pd, const bso_groups* gr, uint32_t a, uint32_t b) {
  const int32_t p1 = pd->priority[a], p2 = pd->priority[b];
  if (p1 != p2) return p1 > p2;
  const int g1 = pd->gid[a], g2 = pd->gid[b];
  const int grouped1 = g1 != BSO_GID_NONE, grouped2 = g2 != BSO_GID_NONE;
  if (grouped1 != grouped2) return grouped1 < grouped2;
  if (!grouped1) return pd->ts_ns[a] < pd->ts_ns[b];
  const int miss1 = g1 < 0 || (uint32_t)g1 >= gr->n || (pd->flags[a] & BSO_POD_LISTER_MISS);
  const int miss2 = g2 < 0 || (uint32_t)g2 >= gr->n || (pd->flags[b] & BSO_POD_LISTER_MISS);
  const int64_t c1 = miss1 ? INT64_MAX : gr->creation_ns[g1];
  const int64_t c2 = miss2 ? INT64_MAX : gr->creation_ns[g2];
  if (c1 != c2) return c1 < c2;
  const uint32_t r1 = miss1 ? 0u : gr->name_rank[g1];
  const uint32_t r2 = miss2 ? 0u : gr->name_rank[g2];
  if (r1 != r2) return r1 > r2;
  return pd->ts_ns[a] < pd->ts_ns[b];
}

static void merge_sort(const bso_pods* pd, const bso_groups* gr, uint32_t* a, uint32_t* tmp,
                       uint32_t n) {
  if (n < 2) return;
  const uint32_t h = n / 2;
  merge_sort(pd, gr, a, tmp, h);
  merge_sort(pd, gr, a + h, tmp, n - h);
  uint32_t i = 0, j = h, k = 0;
  while (i < h && j < n) {
    if (key_less(pd, gr, a[j], a[i])) tmp[k++] = a[j++]; /* stable */
    else tmp[k++] = a[i++];
  }
  while (i < h) tmp[k++] = a[i++];
  while (j < n) tmp[k++] = a[j++];
  memcpy(a, tmp, (size_t)n * sizeof(uint32_t));
}

/* pod x node fit-eval: the composite asserted by core_test.go:108-110,
 * compareResourceAndRequire(singleNodeResource(node,pod,1), getPodResourceRequire(pod)),
 * gated by the callers' node guards (core.go:606-617) and by checkFit itself
 * (an unfit node never hosts the pod; the bare composite would let a pod that
 * requests nothing "fit" a zeroed resource).  score = min over compared lanes
 * of left-req (builder-defined; the reference's Score is a constant, core.go:263). */
int bso_fit_eval(const bso_nodes* nd, const bso_pods* pd, uint32_t p, uint32_t n, int64_t* score) {
  if (score) *score = INT64_MIN;
  if (node_skipped(nd, n)) return 0;
  if (nd->flags[n] & BSO_NODE_TAINTS_ERR) return 0;
  if (!bso_check_fit(nd, n, pd->sel_mask[p], pd->tol_mask[p], POD_AFF(pd, p))) return 0;
  bso_resource left, req;
  bso_single_node_resource(nd, n, pd->sel_mask[p], pd->tol_mask[p], POD_AFF(pd, p), 1.0f, &left);
  bso_pod_require(pd, p, &req);
  if (!bso_compare_resource_and_require(&left, &req, nd->lanes)) return 0;
  if (score) {
    int64_t s = INT64_MAX;
    for (uint32_t d = 0; d < nd->lanes; ++d) {
      if (d >= 4 && !((req.present & left.present) & (1u << d))) continue;
      const int64_t diff = wrap_sub(left.v[d], req.v[d]);
      if (diff < s) s = diff;
    }
    *score = s;
  }
  return 1;
}

/* core.go:436-475 getLeftResource */
int bso_get_left_resource(const bso_nodes* nd, uint32_t n, bso_resource* out) {
  const uint32_t N = nd->n;
  memset(out, 0, sizeof(*out));
  if (nd->flags[n] & BSO_NODE_NIL) return 0;                           /* :447-449 info == nil */
  int64_t pod_count = nd->requested[(size_t)LANE_PODS * N + n];        /* :455-458 */
  if (pod_count == 0) pod_count = nd->pod_count[n];
  out->v[LANE_CPU] = wrap_sub(nd->alloc[(size_t)LANE_CPU * N + n], nd->requested[(size_t)LANE_CPU * N + n]);   /* :460 */
  out->v[LANE_PODS] = wrap_sub(nd->alloc[(size_t)LANE_PODS * N + n], pod_count);                               /* :461 */
  out->v[LANE_MEM] = wrap_sub(nd->alloc[(size_t)LANE_MEM * N + n], nd->requested[(size_t)LANE_MEM * N + n]);   /* :462 */
  out->v[LANE_EPH] = wrap_sub(nd->alloc[(size_t)LANE_EPH * N + n], nd->requested[(size_t)LANE_EPH * N + n]);   /* :463 */
  /* :465-472: leftResourceCopy.ScalarResources is a nil map -> the loop never runs: no scalar keys */
  return 1;
}

/* core.go:514-564 computeResourceSatisfied (Filter, :170-191, maps its error) */
int bso_filter_eval(const bso_nodes* nd, const bso_pods* pd, uint32_t p, uint32_t n, int m, int max_has_minres,
                    const bso_resource* max_min_res) {
  const int g = pd->gid[p];
  if (g == BSO_GID_NONE) return BSO_FILTER_PASS;                       /* :171-174 */
  if (g < 0) return BSO_FILTER_NOT_FOUND;                              /* :177-180 */
  if (m < 0) return BSO_FILTER_REF_PANIC;                              /* :525 sop.maxPGStatus == nil */
  if (m == g) return BSO_FILTER_PASS;                                  /* :531-535 case 1 */
  if (!max_has_minres) return BSO_FILTER_PASS;                         /* :542-544 */
  bso_resource left, req;
  if (!bso_get_left_resource(nd, n, &left)) return BSO_FILTER_NO_SNAPSHOT;   /* :545-548 */
  bso_pod_require(pd, p, &req);                                        /* :551 */
  bso_resource_add(&req, max_min_res, nd->lanes);                      /* :552 */
  if (bso_compare_resource_and_require(&left, &req, nd->lanes)) return BSO_FILTER_PASS;          /* :553 case 2 */
  if (!bso_compare_resource_and_require(&left, max_min_res, nd->lanes)) return BSO_FILTER_PASS;  /* :558 case 3 */
  return BSO_FILTER_NOT_ENOUGH;                                        /* :563 */
}

/* ------------------------------------------------------------------------ */
/* Effective group state of a round: what fillOccupiedObj (core.go:477-512)
 * leaves behind once the first pod of each group (table order) has reached it:
 * pgs.Pod (:486-488) and the MinResources default (:489-493).  A pod reaches
 * fillOccupiedObj only if it is grouped, not recently permitted (:95-98), its
 * group exists (:100-103) and is not in the deny cache (:105-110). */
typedef struct {
  uint8_t* flags;
  uint64_t* rep_sel;
  uint64_t* rep_tol;
  uint32_t* rep_aff;
  int64_t* min_res; /* [lanes][G] */
  uint32_t* min_res_present;
} eff_groups;

static int reaches_fill(const bso_pods* pd, const bso_groups* gr, uint32_t p) {
  const int g = pd->gid[p];
  if (g < 0 || (uint32_t)g >= gr->n) return 0;
  if (pd->flags[p] & BSO_POD_PERMITTED_RECENTLY) return 0;
  if (gr->flags[g] & BSO_GROUP_DENIED) return 0;
  return 1;
}

static void fill_from_pod(const bso_pods* pd, const bso_groups* gr, eff_groups* eg, uint32_t p) {
  const uint32_t g = (uint32_t)pd->gid[p];
  if (!(eg->flags[g] & BSO_GROUP_HAS_POD)) { /* :486-488 */
    eg->flags[g] |= BSO_GROUP_HAS_POD;
    eg->rep_sel[g] = pd->sel_mask[p];
    eg->rep_tol[g] = pd->tol_mask[p];
    eg->rep_aff[g] = POD_AFF(pd, p);
  }
  if (!(eg->flags[g] & BSO_GROUP_HAS_MINRES)) { /* :489-493 */
    eg->flags[g] |= BSO_GROUP_HAS_MINRES;
    for (uint32_t d = 0; d < gr->lanes; ++d) {
      const int pres = d < 4 || (pd->req_present[p] & (1u << d));
      eg->min_res[(size_t)d * gr->n + g] = pres ? pd->req[(size_t)d * pd->n + p] : 0;
    }
    eg->min_res_present[g] = pd->req_present[p] & ~0xFu;
  }
}

static int eff_alloc(const bso_groups* gr, eff_groups* eg) {
  const size_t G = gr->n ? gr->n : 1;
  eg->flags = (uint8_t*)malloc(G);
  eg->rep_sel = (uint64_t*)malloc(G * 8);
  eg->rep_tol = (uint64_t*)malloc(G * 8);
  eg->rep_aff = (uint32_t*)malloc(G * 4);
  eg->min_res = (int64_t*)malloc(G * 8 * gr->lanes);
  eg->min_res_present = (uint32_t*)malloc(G * 4);
  if (!eg->flags || !eg->rep_sel || !eg->rep_tol || !eg->rep_aff || !eg->min_res || !eg->min_res_present) return -1;
  memcpy(eg->flags, gr->flags, gr->n);
  memcpy(eg->rep_sel, gr->rep_sel, (size_t)gr->n * 8);
  memcpy(eg->rep_tol, gr->rep_tol, (size_t)gr->n * 8);
  for (uint32_t g = 0; g < gr->n; ++g) eg->rep_aff[g] = gr->rep_aff ? gr->rep_aff[g] : BSO_AFF_NONE;
  memcpy(eg->min_res, gr->min_res, (size_t)gr->n * 8 * gr->lanes);
  memcpy(eg->min_res_present, gr->min_res_present, (size_t)gr->n * 4);
  return 0;
}

static void eff_free(eff_groups* eg) {
  free(eg->flags); free(eg->rep_sel); free(eg->rep_tol); free(eg->rep_aff); free(eg->min_res);
  free(eg->min_res_present);
}

static void eff_pre_allocated(const bso_groups* gr, const eff_groups* eg, uint32_t g,
                              int64_t matched, bso_resource* out) {
  int64_t mr[BSO_MAX_LANES];
  for (uint32_t d = 0; d < gr->lanes; ++d) mr[d] = eg->min_res[(size_t)d * gr->n + g];
  pre_allocated_cols(gr, g, matched, (eg->flags[g] & BSO_GROUP_HAS_MINRES) != 0, mr,
                     eg->min_res_present[g], out);
}

/* core.go:88-167 PreFilter for one pod against the frozen round state.
 * m / max_matched: findMaxPG result (recomputed by the caller per pod when
 * faithful).  Sets *deny when the group is added to the deny cache (:142,163). */
static uint8_t prefilter_one(const bso_nodes* nd, const bso_pods* pd, const bso_groups* gr,
                             const eff_groups* eg, uint32_t p, int m, int* deny) {
  *deny = 0;
  const int g = pd->gid[p];
  if (g == BSO_GID_NONE) return BSO_PF_PASS;                          /* :89-92 */
  if (pd->flags[p] & BSO_POD_PERMITTED_RECENTLY) return BSO_PF_PASS;  /* :95-98 */
  if (g < 0 || (uint32_t)g >= gr->n) return BSO_PF_NOT_FOUND;         /* :100-103 */
  if (gr->flags[g] & BSO_GROUP_DENIED) return BSO_PF_DENIED;          /* :105-110 */
  if (pd->flags[p] & BSO_POD_OCC_NOREFS) return BSO_PF_OCC_NOREFS;    /* :504-506 */
  if (pd->flags[p] & BSO_POD_OCC_MISMATCH) return BSO_PF_OCCUPIED;    /* :507-510 */
  if (m < 0) return BSO_PF_PASS;                                      /* :127-130 */
  const uint32_t matched = gr->matched[m];                            /* :132-135 */
  bso_resource need, req;
  if (matched == 0) {                                                 /* :136 */
    eff_pre_allocated(gr, eg, (uint32_t)g, 0, &need);                 /* :137-139 own group */
    if (!bso_compare_cluster(nd, eg->rep_sel[g], eg->rep_tol[g], eg->rep_aff[g], &need, 1.0f)) { /* :140 */
      *deny = 1;                                                      /* :142 */
      return BSO_PF_NOT_ENOUGH;                                       /* :143 */
    }
    return BSO_PF_PASS;                                               /* :146 */
  }
  if (m == g) return BSO_PF_PASS;                                     /* :150-155 */
  eff_pre_allocated(gr, eg, (uint32_t)m, (int64_t)matched, &need);    /* :157 */
  bso_pod_require(pd, p, &req);                                       /* :158 */
  bso_resource_add(&need, &req, nd->lanes);                           /* :159 */
  if (!bso_compare_cluster(nd, eg->rep_sel[m], eg->rep_tol[m], eg->rep_aff[m], &need, 0.7f)) { /* :161 */
    *deny = 1;                                                        /* :163 */
    return BSO_PF_NOT_ENOUGH;                                         /* :164 */
  }
  return BSO_PF_PASS;
}

int bso_round(const bso_nodes* nd, const bso_pods* pd, const bso_groups* gr, bso_results* out,
              int faithful, int threads) {
  const uint32_t P = pd->n, N = nd->n, G = gr->n;
  const uint32_t words = (N + 31) / 32;
  eff_groups eg;
  if (eff_alloc(gr, &eg)) return -1;
#ifdef _OPENMP
  if (threads <= 0) threads = omp_get_max_threads();
#else
  threads = 1;
#endif
  (void)threads;

  /* D.1: first-pod capture, in table order */
  for (uint32_t p = 0; p < P; ++p)
    if (reaches_fill(pd, gr, p)) fill_from_pod(pd, gr, &eg, p);

  /* D.2: findMaxPG once per round over the effective flags */
  int panic = 0;
  uint32_t max_fin = 0;
  int m = find_max_pg_flags(gr, eg.flags, &max_fin, &panic);
  out->max_group = m;
  out->max_finished = max_fin;
  out->ref_panic = panic;
  if (panic) { eff_free(&eg); return 1; }

  if (out->new_denied) memset(out->new_denied, 0, G);
  uint8_t* pf = out->prefilter;
  uint8_t* denied_tmp = (uint8_t*)calloc(G ? G : 1, 1);

  /* per-group cache for the matched==0 branch when not faithful:
   * 0 unknown, 1 ok, 2 not enough */
  uint8_t* gcache = (uint8_t*)calloc(G ? G : 1, 1);

#pragma omp parallel for schedule(dynamic, 64) num_threads(threads)
  for (uint32_t p = 0; p < P; ++p) {
    int deny = 0;
    uint8_t code;
    if (faithful) {
      /* the reference recomputes findMaxPG for every pod (core.go:119-123) */
      uint32_t mf;
      int pn;
      int m2 = find_max_pg_flags(gr, eg.flags, &mf, &pn);
      code = prefilter_one(nd, pd, gr, &eg, p, m2, &deny);
    } else {
      const int g = pd->gid[p];
      int cached = 0;
      if (m >= 0 && gr->matched[m] == 0 && g >= 0 && (uint32_t)g < G) {
        uint8_t c;
#pragma omp atomic read
        c = gcache[g];
        if (c && reaches_fill(pd, gr, p) &&
            !(pd->flags[p] & (BSO_POD_OCC_NOREFS | BSO_POD_OCC_MISMATCH))) {
          code = (c == 1) ? BSO_PF_PASS : BSO_PF_NOT_ENOUGH;
          deny = (c == 2);
          cached = 1;
        }
      }
      if (!cached) {
        code = prefilter_one(nd, pd, gr, &eg, p, m, &deny);
        if (m >= 0 && gr->matched[m] == 0 && g >= 0 && (uint32_t)g < G &&
            (code == BSO_PF_PASS || code == BSO_PF_NOT_ENOUGH) && reaches_fill(pd, gr, p) &&
            !(pd->flags[p] & (BSO_POD_OCC_NOREFS | BSO_POD_OCC_MISMATCH))) {
          uint8_t c = (code == BSO_PF_PASS) ? 1 : 2;
#pragma omp atomic write
          gcache[g] = c;
          (void)c;
        }
      }
    }
    if (pf) pf[p] = code;
    if (deny) {
#pragma omp atomic write
      denied_tmp[pd->gid[p]] = 1;
    }
  }
  if (out->new_denied) memcpy(out->new_denied, denied_tmp, G);
  free(gcache);

  /* D.3: pod x node fit-evals with the pod's own masks at percent 1.0 */
  uint32_t* contrib = (uint32_t*)calloc(G ? G : 1, sizeof(uint32_t));
  uint32_t* in_round = (uint32_t*)calloc(G ? G : 1, sizeof(uint32_t));
  uint8_t* any_fit = (uint8_t*)calloc(P ? P : 1, 1);
#pragma omp parallel for schedule(dynamic, 16) num_threads(threads)
  for (uint32_t p = 0; p < P; ++p) {
    uint32_t cnt = 0;
    int32_t best = -1;
    int64_t best_s = INT64_MIN;
    uint32_t* row = out->fit_bitmap ? out->fit_bitmap + (size_t)p * words : NULL;
    int64_t* srow = out->score ? out->score + (size_t)p * N : NULL;
    if (row) memset(row, 0, (size_t)words * 4);
    for (uint32_t n = 0; n < N; ++n) {
      int64_t s;
      const int f = bso_fit_eval(nd, pd, p, n, &s);
      if (srow) srow[n] = s;
      if (f) {
        ++cnt;
        if (row) row[n >> 5] |= 1u << (n & 31);
        if (best < 0 || s > best_s) { best = (int32_t)n; best_s = s; }
      }
    }
    if (out->feasible_count) out->feasible_count[p] = cnt;
    if (out->best_node) out->best_node[p] = best;
    if (out->best_score) out->best_score[p] = best_s;
    any_fit[p] = cnt > 0;
  }

  /* Filter (SURVEY 8(f) row 2): computeResourceSatisfied per (pod,node) against the round's max group */
  if (out->filter_bitmap || out->filter_code) {
    bso_resource mmr;
    memset(&mmr, 0, sizeof(mmr));
    int has_mr = 0;
    if (m >= 0 && (eg.flags[m] & BSO_GROUP_HAS_MINRES)) {
      has_mr = 1;   /* :525-528: Resource{}.Add(*MinResources) */
      for (uint32_t d = 0; d < gr->lanes; ++d) {
        if (d >= 4 && !(eg.min_res_present[m] & (1u << d))) continue;
        mmr.v[d] = eg.min_res[(size_t)d * G + m];
      }
      mmr.present = eg.min_res_present[m];
    }
#pragma omp parallel for schedule(dynamic, 16) num_threads(threads)
    for (uint32_t p = 0; p < P; ++p) {
      uint32_t* row = out->filter_bitmap ? out->filter_bitmap + (size_t)p * words : NULL;
      if (row) memset(row, 0, (size_t)words * 4);
      const int g = pd->gid[p];
      uint8_t pcode = BSO_FILTER_PASS;
      if (g != BSO_GID_NONE && (g < 0 || (uint32_t)g >= G)) pcode = BSO_FILTER_NOT_FOUND;
      else if (g != BSO_GID_NONE && m < 0) pcode = BSO_FILTER_REF_PANIC;
      if (out->filter_code) out->filter_code[p] = pcode;
      if (!row) continue;
      for (uint32_t n = 0; n < N; ++n) {
        const int gg = (g >= 0 && (uint32_t)g >= G) ? BSO_GID_MISSING : g;
        bso_pods pd2 = *pd;
        (void)pd2;
        int c;
        if (gg == BSO_GID_MISSING) c = BSO_FILTER_NOT_FOUND;
        else c = bso_filter_eval(nd, pd, p, n, m, has_mr, &mmr);
        if (c == BSO_FILTER_PASS) row[n >> 5] |= 1u << (n & 31);
      }
    }
  }

  /* D.4: Permit readiness per group (core.go:303) */
  for (uint32_t p = 0; p < P; ++p) {
    const int g = pd->gid[p];
    if (g < 0 || (uint32_t)g >= G) continue;
    in_round[g]++;
    const uint8_t code = pf ? pf[p] : BSO_PF_PASS;
    if (code == BSO_PF_PASS && any_fit[p]) contrib[g]++;
  }
  if (out->admit_bitmap) memset(out->admit_bitmap, 0, (size_t)((G + 31) / 32) * 4);
  for (uint32_t g = 0; g < G; ++g) {
    const uint32_t cnt = gr->matched[g] + contrib[g];
    uint8_t a;
    if (in_round[g] > 0 && contrib[g] == 0) a = BSO_UNSCHEDULABLE;
    else a = bso_permit_ready(cnt, gr->min_member[g], gr->scheduled[g]) ? BSO_ADMIT : BSO_WAIT;
    if (out->admit) out->admit[g] = a;
    if (a == BSO_ADMIT && out->admit_bitmap) out->admit_bitmap[g >> 5] |= 1u << (g & 31);
  }

  /* D.5: queue order */
  if (out->order || out->rank) {
    uint32_t* ord = (uint32_t*)malloc((size_t)(P ? P : 1) * 4);
    uint32_t* tmp = (uint32_t*)malloc((size_t)(P ? P : 1) * 4);
    for (uint32_t p = 0; p < P; ++p) ord[p] = p;
    merge_sort(pd, gr, ord, tmp, P);
    if (out->order) memcpy(out->order, ord, (size_t)P * 4);
    if (out->rank) {
      uint32_t r = 0;
      for (uint32_t i = 0; i < P; ++i) {
        if (i > 0 && (key_less(pd, gr, ord[i - 1], ord[i]) || key_less(pd, gr, ord[i], ord[i - 1]))) ++r;
        out->rank[ord[i]] = r;
      }
    }
    free(ord); free(tmp);
  }

  free(contrib); free(in_round); free(any_fit); free(denied_tmp);
  eff_free(&eg);
  return 0;
}

/* ------------------------------------------------------------------------ */
/* Sequential replay: the reference's pod-at-a-time cycle with mutable state. */
int bso_replay(bso_nodes* nd, const bso_pods* pd, bso_groups* gr, const uint32_t* queue,
               uint32_t n_queue, uint8_t* prefilter_out, int32_t* node_out, uint8_t* ready_out) {
  const uint32_t N = nd->n, L = nd->lanes;
  int panic_at = -1;
  for (uint32_t qi = 0; qi < n_queue; ++qi) {
    const uint32_t p = queue[qi];
    const int g = pd->gid[p];
    prefilter_out[qi] = BSO_PF_PASS;
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
      if (pn && panic_at < 0) panic_at = (int)qi;
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
    /* ---- stand-in for the upstream filter/selectHost: first fitting node ---- */
    int32_t chosen = -1;
    for (uint32_t n = 0; n < N; ++n)
      if (bso_fit_eval(nd, pd, p, n, NULL)) { chosen = (int32_t)n; break; }
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
    /* ---- Permit, core.go:268-309 ---- */
    if (g < 0 || (uint32_t)g >= gr->n) { ready_out[qi] = 1; continue; }
    gr->matched[g] += 1; /* :290 MatchedPodNodes.Set */
    if (bso_permit_ready(gr->matched[g], gr->min_member[g], gr->scheduled[g])) {
      gr->flags[g] |= BSO_GROUP_SCHEDULED; /* :305 */
      ready_out[qi] = 1;
    }
  }
  return panic_at;
}
