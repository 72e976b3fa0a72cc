/*
 * bs_oracle.h — TEST INFRASTRUCTURE, NOT PRODUCT.
 *
 * CPU restatement (plain C) of the PreFilter / Permit / Compare hot path of
 * tenstack/batch-scheduler, pkg/scheduler/core/core.go.  Only tests/,
 * __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs
 * may link or call this.  The product (batch-scheduler_b200/csrc) never does.
 *
 * The reference is Go and needs k8s.io/kubernetes v1.17.5 + ~130 modules that
 * are not on disk, and there is no Go toolchain here, so the reference itself
 * cannot be built (oracle/_ref does not exist).  What pins this restatement:
 *   - the reference's own test, pkg/scheduler/core/core_test.go:27-115 (3 cases);
 *   - the README resource-race scenario, README.md:76-188 (one gang admitted);
 *   - float32 scaling vectors computed independently with numpy.float32.
 * Everything else on the path (findMaxPG, the 0.7 factor, the early-exit scan,
 * getPreAllocatedResource, Permit, Compare, deny cache) has NO reference test:
 * for those rows parity is UNPINNED by the reference and rests on this file
 * following core.go line by line.  Third-party arithmetic restated from its
 * published behaviour (source absent): k8s.io/kubernetes v1.17.5
 * pkg/scheduler/nodeinfo Resource.Add / ResourceList (int64 field sums through
 * an exact resource.Quantity round trip), predicates.PodMatchNodeSelector /
 * PodToleratesNodeTaints (pre-encoded as bitmasks by the packer).
 */
#ifndef BS_ORACLE_H
#define BS_ORACLE_H
#include <stdint.h>

#define BSO_MAX_LANES 16

/* flag values are the same as include/bsched.h (checked by tests/test_abi.py) */
#define BSO_NODE_NIL 0x01u
#define BSO_NODE_NO_NODE 0x02u
#define BSO_NODE_UNSCHEDULABLE 0x04u
#define BSO_NODE_TAINTS_ERR 0x08u
#define BSO_POD_PERMITTED_RECENTLY 0x01u
#define BSO_POD_OCC_NOREFS 0x02u
#define BSO_POD_OCC_MISMATCH 0x04u
#define BSO_POD_LISTER_MISS 0x08u
#define BSO_GROUP_SCHEDULED 0x01u
#define BSO_GROUP_HAS_POD 0x02u
#define BSO_GROUP_HAS_MINRES 0x04u
#define BSO_GROUP_DENIED 0x08u
#define BSO_AFF_NONE 0xffffffffu
#define BSO_GID_NONE (-1)
#define BSO_GID_MISSING (-2)

enum { BSO_PF_PASS = 0, BSO_PF_NOT_FOUND = 1, BSO_PF_DENIED = 2, BSO_PF_OCC_NOREFS = 3,
       BSO_PF_OCCUPIED = 4, BSO_PF_NOT_ENOUGH = 5 };
enum { BSO_ADMIT = 0, BSO_WAIT = 1, BSO_UNSCHEDULABLE = 2 };
/* Filter verdict per (pod,node), core.go:170-191 + computeResourceSatisfied :514-564 */
enum { BSO_FILTER_PASS = 0, BSO_FILTER_NOT_FOUND = 1, BSO_FILTER_NOT_ENOUGH = 2, BSO_FILTER_NO_SNAPSHOT = 3,
       BSO_FILTER_REF_PANIC = 4 };

/* nodeinfo.Resource: 4 fixed fields + ScalarResources map (key presence = bit) */
typedef struct {
  int64_t v[BSO_MAX_LANES];
  uint32_t present;
} bso_resource;

typedef struct {
  uint32_t n, lanes;
  int64_t* alloc;      /* [lanes][n] */
  int64_t* requested;  /* [lanes][n] */
  int32_t* pod_count;
  uint32_t* alloc_present;
  uint32_t* req_present;
  uint64_t* label_mask;
  uint64_t* taint_mask;
  uint8_t* flags;
  uint32_t n_aff;      /* affinity classes in aff_bits (0: none) */
  uint32_t* aff_bits;  /* [n_aff][ceil(n/32)] host-evaluated (affinity class, node) predicate bits, or NULL */
} bso_nodes;

typedef struct {
  uint32_t n, lanes;
  int64_t* req; /* [lanes][n] */
  uint32_t* req_present;
  int32_t* gid;
  uint64_t* sel_mask;
  uint64_t* tol_mask;
  int32_t* priority;
  int64_t* ts_ns;
  uint8_t* flags;
  uint32_t* aff_class; /* [n] row of aff_bits the pod must match, BSO_AFF_NONE = none; NULL = all NONE */
} bso_pods;

typedef struct {
  uint32_t n, lanes;
  uint32_t* min_member;
  uint32_t* scheduled;
  uint32_t* matched;
  uint8_t* flags;
  int64_t* min_res; /* [lanes][n] */
  uint32_t* min_res_present;
  uint64_t* rep_sel;
  uint64_t* rep_tol;
  int64_t* creation_ns;
  uint32_t* name_rank;
  uint32_t* rep_aff;   /* affinity class of pgs.Pod, or NULL */
} bso_groups;

typedef struct {
  uint8_t* prefilter;        /* [P] */
  uint32_t* feasible_count;  /* [P] */
  int32_t* best_node;        /* [P] */
  int64_t* best_score;       /* [P] */
  uint8_t* admit;            /* [G] */
  uint32_t* admit_bitmap;    /* [ceil(G/32)] */
  uint8_t* new_denied;       /* [G] */
  uint32_t* order;           /* [P] */
  uint32_t* rank;            /* [P] */
  uint32_t* filter_bitmap;   /* [P][ceil(N/32)] bit = Filter passes, or NULL */
  uint8_t* filter_code;      /* [P] pod-level Filter outcome when it does not depend on the node */
  uint32_t* fit_bitmap;      /* [P][ceil(N/32)] or NULL */
  int64_t* score;            /* [P][N] or NULL */
  int32_t max_group;
  uint32_t max_finished;
  int32_t ref_panic;         /* 1: findMaxPG would divide by zero */
} bso_results;

/* ---- line-by-line helpers ---- */
int64_t bso_scale(int64_t alloc, float percent);                              /* core.go:656-659,667 */
int bso_check_fit(const bso_nodes* nd, uint32_t i, uint64_t sel, uint64_t tol, uint32_t aff); /* core.go:741-759 */
void bso_single_node_resource(const bso_nodes* nd, uint32_t i, uint64_t sel, uint64_t tol, uint32_t aff,
                              float percent, bso_resource* out);              /* core.go:634-670 */
int bso_compare_resource_and_require(const bso_resource* left, const bso_resource* req,
                                     uint32_t lanes);                         /* core.go:672-699 */
void bso_resource_add(bso_resource* acc, const bso_resource* x, uint32_t lanes); /* Resource.Add(x.ResourceList()) */
int bso_compare_cluster(const bso_nodes* nd, uint64_t sel, uint64_t tol, uint32_t aff, const bso_resource* need,
                        float percent);                                       /* core.go:595-632 */
void bso_compute_cluster(const bso_nodes* nd, uint64_t sel, uint64_t tol, uint32_t aff, bso_resource* out); /* core.go:566-593 */
int bso_find_max_pg(const bso_groups* gr, uint32_t* max_finished, int* panic); /* core.go:701-739 */
void bso_pre_allocated(const bso_groups* gr, uint32_t g, int64_t matched, bso_resource* out); /* core.go:774-793 */
void bso_pod_require(const bso_pods* pd, uint32_t p, bso_resource* out);      /* core.go:761-772 (packed) */
int bso_permit_ready(uint32_t matched_count, uint32_t min_member, uint32_t scheduled); /* core.go:303 */
int bso_compare(const bso_pods* pd, const bso_groups* gr, uint32_t a, uint32_t b); /* core.go:368-411 */
int bso_fit_eval(const bso_nodes* nd, const bso_pods* pd, uint32_t p, uint32_t n, int64_t* score);
/* getLeftResource (core.go:436-475): plain alloc - requested, no float32 factor, no checkFit, and
 * never any scalar key (the Clone of a zero Resource has a nil map, :465-472).  Returns 0 when the
 * reference returns nil (info == nil). */
int bso_get_left_resource(const bso_nodes* nd, uint32_t n, bso_resource* out);
/* computeResourceSatisfied (core.go:514-564) for one (pod,node) given the round's max group m and its
 * effective MinResources; returns a BSO_FILTER_* code. */
int bso_filter_eval(const bso_nodes* nd, const bso_pods* pd, uint32_t p, uint32_t n, int m, int max_has_minres,
                    const bso_resource* max_min_res);

/* ---- one snapshot round (SURVEY.md Appendix D; DESIGN.md "Round semantics") ----
 * faithful != 0: PreFilter is evaluated the way the reference does it, per pod:
 * findMaxPG over all groups and the ordered node scan are re-run for every pod
 * (core.go:120,140,161).  faithful == 0: same results, shared work hoisted.
 * threads: OpenMP threads for the per-pod loops (<=0: all). */
int bso_round(const bso_nodes* nd, const bso_pods* pd, const bso_groups* gr, bso_results* out,
              int faithful, int threads);

/* ---- sequential replay of the reference's pod-at-a-time cycle (README scenario) ----
 * Pods are processed in queue order; state (requested, pod_count, matched,
 * scheduled, flags) is mutated in place like the reference's caches.  A pod that
 * passes PreFilter is assumed onto the first node (list order) where it fits.
 * prefilter_out[P], node_out[P] (-1 none), ready_out[P].  Returns the first queue position whose findMaxPG would
 * divide by MinMember == 0 (core.go:716, where the reference panics), or -1; the walk goes on past it as if that group
 * were left out, so every output is as without the check. */
int bso_replay(bso_nodes* nd, const bso_pods* pd, bso_groups* gr, const uint32_t* queue,
               uint32_t n_queue, uint8_t* prefilter_out, int32_t* node_out, uint8_t* ready_out);

/* ---- state around Permit (bs_gang.c): the reference's go-cache TTL tables, restated from their call sites ---- */
typedef struct bso_gang bso_gang;
bso_gang* bso_gang_new(uint32_t n_groups);
void bso_gang_free(bso_gang* s);
int bso_permit_step(bso_gang* s, uint32_t g, uint64_t uid, uint64_t name, uint32_t node, int64_t now, int64_t wait_ns,
                    uint32_t min_member, uint32_t scheduled);                        /* core.go:283-307 */
uint32_t bso_expire(bso_gang* s, int64_t now, uint32_t* rej_group, uint64_t* rej_uid, uint32_t cap, uint32_t* evicted,
                    uint32_t ecap, uint32_t* n_evicted);                             /* controller.go:322-333 */
uint32_t bso_allow_list(bso_gang* s, uint32_t g, int64_t now, uint32_t min_member, uint32_t scheduled, uint64_t* uids,
                        uint32_t* nodes, uint32_t cap);                              /* batchscheduler.go:292-344 */
uint32_t bso_gang_matched(const bso_gang* s, uint32_t g, int64_t now);
int bso_gang_scheduled(const bso_gang* s, uint32_t g);
int bso_gang_denied(bso_gang* s, uint32_t g, int64_t now);
void bso_gang_deny(bso_gang* s, uint32_t g, int64_t now);                            /* core.go:423-425 */
int bso_gang_permitted(bso_gang* s, uint64_t uid, int64_t now);
void bso_gang_mark_permitted(bso_gang* s, uint64_t uid, int64_t now);                /* core.go:188 */

int bso_max_threads(void);
#endif
