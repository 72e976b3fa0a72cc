/*
 * bsched.h — C ABI of the H100 gang-scheduling feasibility engine.
 *
 * This is the drop-in boundary for the PreFilter / Permit / Less hot path of
 * tenstack/batch-scheduler.  Every entry point names the reference interface it
 * replaces (paths are relative to the reference repository root).  The Go side
 * binds these through cgo (see INTEGRATION.md); Python binds them through ctypes
 * (batch-scheduler_b200/capi.py); nothing but plain pointers and sizes crosses.
 *
 * Conventions
 *   - every function returns 0 (BS_OK) or a negative bs_err; nothing aborts;
 *   - the caller owns every input array for the duration of the call only
 *     (cgo rule: no Go pointer is retained); the engine owns device memory;
 *   - outputs are written into caller-provided buffers;
 *   - a handle is thread-safe: calls on one bs_engine serialise on an internal
 *     mutex (the reference calls Less/Permit from several goroutines,
 *     pkg/scheduler/batch/batchscheduler.go:165,214);
 *   - there is NO CPU fallback: without a CUDA device bs_create fails with
 *     BS_E_NODEVICE.
 *
 * Resource lanes (SoA, int64): lane 0 MilliCPU, 1 Memory, 2 EphemeralStorage,
 * 3 AllowedPodNumber (the four fixed nodeinfo.Resource fields used at
 * pkg/scheduler/core/core.go:656-659,673-685), lanes 4.. are the scalar /
 * extended resources (`ScalarResources`, core.go:662-668,686-697).  Map-key
 * presence of a scalar resource is a bit in a uint32 mask (bit d = lane d).
 * Tables are lane-major: value of lane d for row i is a[d * n_rows + i].
 */
#ifndef BSCHED_H
#define BSCHED_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BS_ABI_VERSION 8
#define BS_FIXED_LANES 4
#define BS_MAX_LANES 16
/* |value| bound accepted for every int64 table entry (validated at upload):
 * keeps left-req differences and the float32->int64 conversion in range. */
#define BS_VALUE_LIMIT ((int64_t)1 << 56)

typedef struct bs_engine bs_engine; /* opaque */

typedef enum {
  BS_OK = 0,
  BS_E_INVAL = -1,       /* bad argument / table shape */
  BS_E_NODEVICE = -2,    /* no CUDA device: there is no CPU path */
  BS_E_CUDA = -3,        /* CUDA runtime error (bs_last_error has the text) */
  BS_E_NOMEM = -4,
  BS_E_RANGE = -5,       /* table value outside +-BS_VALUE_LIMIT */
  BS_E_STATE = -6,       /* call out of order (e.g. evaluate before upload) */
  BS_E_REF_PANIC = -7,   /* the reference would panic on this input:
                            findMaxPG divides by MinMember==0 (core.go:716-717) */
  BS_E_INDEX = -8,       /* pod / node / group index out of range */
  BS_E_PEER = -9         /* peer exchange timed out (a rank did not arrive) */
} bs_err;

/* ---- framework.Status codes (k8s.io/kubernetes v1.17.5
 *      pkg/scheduler/framework/v1alpha1; the adapter maps onto them at
 *      batchscheduler.go:104-107,183-201) ---- */
typedef enum {
  BS_CODE_SUCCESS = 0,
  BS_CODE_ERROR = 1,
  BS_CODE_UNSCHEDULABLE = 2,
  BS_CODE_UNSCHEDULABLE_AND_UNRESOLVABLE = 3,
  BS_CODE_WAIT = 4,
  BS_CODE_SKIP = 5
} bs_code;

/* ---- PreFilter verdict per pod (reason enum -> message, core.go:88-167) ---- */
typedef enum {
  BS_PF_PASS = 0,
  BS_PF_ERR_NOT_FOUND = 1,   /* "can not found pod group: %v"          core.go:102 */
  BS_PF_ERR_DENIED = 2,      /* "pod with pgName: %v last failed in 20s, deny" :107 */
  BS_PF_ERR_OCCUPIED_NOREFS = 3, /* "pod group %s has been occupied by %v"   :505 */
  BS_PF_ERR_OCCUPIED = 4,    /* "pod group has been occupied by %v"          :509 */
  BS_PF_ERR_NOT_ENOUGH = 5   /* "cluster resource not enough"           :143,:164 */
} bs_prefilter_code;

/* ---- Filter verdict (core.go:170-191 + computeResourceSatisfied :514-564) ---- */
typedef enum {
  BS_FILTER_PASS = 0,
  BS_FILTER_ERR_NOT_FOUND = 1,   /* "can not found pod group: %v" (bare pgName)   core.go:179 */
  BS_FILTER_ERR_NOT_ENOUGH = 2,  /* util.ErrorResourceNotEnough "resource not enough"    :563 */
  BS_FILTER_ERR_NO_SNAPSHOT = 3, /* "SnapShot not initialized"                           :547 */
  BS_FILTER_REF_PANIC = 4        /* sop.maxPGStatus == nil is dereferenced at            :525 */
} bs_filter_code;

/* ---- gang decision per group (Permit, core.go:268-309) ---- */
typedef enum {
  BS_ADMIT = 0,         /* ready: matched >= MinMember - Status.Scheduled (uint32) */
  BS_WAIT = 1,          /* not ready yet -> framework.Wait                         */
  BS_UNSCHEDULABLE = 2  /* pods in the round, none passed PreFilter with a node    */
} bs_admit_code;

/* ---- node flags: the guards of core.go:606-617 and :639 ---- */
#define BS_NODE_NIL 0x01u           /* info == nil                   core.go:606 */
#define BS_NODE_NO_NODE 0x02u       /* info.Node() == nil            core.go:610 */
#define BS_NODE_UNSCHEDULABLE 0x04u /* Spec.Unschedulable            core.go:615 */
#define BS_NODE_TAINTS_ERR 0x08u    /* info.Taints() returned error  core.go:639 */

/* ---- pod flags ---- */
#define BS_POD_PERMITTED_RECENTLY 0x01u /* uid in lastPermittedPod   core.go:95-98 */
#define BS_POD_OCC_NOREFS 0x02u   /* group occupied, pod has no ownerRefs  :504-506 */
#define BS_POD_OCC_MISMATCH 0x04u /* group occupied by other owner refs    :507-510 */
#define BS_POD_LISTER_MISS 0x08u  /* pgLister.Get fails for this pod       :395-399 */

/* ---- group flags (cache.PodGroupMatchStatus, pkg/scheduler/cache/cache.go:52-67) ---- */
#define BS_GROUP_SCHEDULED 0x01u   /* pgs.Scheduled                cache.go:66 */
#define BS_GROUP_HAS_POD 0x02u     /* pgs.Pod != nil               cache.go:64 */
#define BS_GROUP_HAS_MINRES 0x04u  /* Spec.MinResources != nil     types.go:97 */
#define BS_GROUP_DENIED 0x08u      /* ns/name in lastDeniedPG      core.go:105 */

/* affinity class of a pod / a group's representative pod: BS_AFF_NONE = no constraint beyond the masks */
#define BS_AFF_NONE 0xffffffffu

/* gid values for pods that carry no usable group */
#define BS_GID_NONE (-1)    /* no group label: VerifyPodLabelSatisfied false (k8s.go:62) */
#define BS_GID_MISSING (-2) /* labelled, but podGroupStatusCache.Get == nil (core.go:100) */

/* Node table: the scheduler snapshot, in snapshot LIST ORDER (core.go:597,604). */
typedef struct {
  uint32_t n_nodes;
  uint32_t n_lanes;              /* 4..BS_MAX_LANES, same for all three tables */
  const int64_t* alloc;          /* [n_lanes][n_nodes] info.AllocatableResource() */
  const int64_t* requested;      /* [n_lanes][n_nodes] info.RequestedResource()   */
  const int32_t* pod_count;      /* [n_nodes] len(info.Pods())        core.go:650-653 */
  const uint32_t* alloc_present; /* [n_nodes] scalar keys in allocatable          */
  const uint32_t* req_present;   /* [n_nodes] scalar keys in requested            */
  const uint64_t* label_mask;    /* [n_nodes] pre-encoded node labels (checkFit, core.go:741) */
  const uint64_t* taint_mask;    /* [n_nodes] pre-encoded NoSchedule/NoExecute taints */
  const uint8_t* flags;          /* [n_nodes] BS_NODE_* */
} bs_node_table;

/* Pod table: the queue candidates of one round. */
typedef struct {
  uint32_t n_pods;
  uint32_t n_lanes;
  const int64_t* req;          /* [n_lanes][n_pods] getPodResourceRequire  core.go:761-772 */
  const uint32_t* req_present; /* [n_pods] scalar keys present in the request            */
  const int32_t* gid;          /* [n_pods] group index, BS_GID_NONE or BS_GID_MISSING    */
  const uint64_t* sel_mask;    /* [n_pods] required node-label bits                      */
  const uint64_t* tol_mask;    /* [n_pods] tolerated taint bits                          */
  const int32_t* priority;     /* [n_pods] podutil.GetPodPriority         core.go:372    */
  const int64_t* ts_ns;        /* [n_pods] PodInfo.Timestamp              core.go:385    */
  const uint8_t* flags;        /* [n_pods] BS_POD_*                                      */
  const uint32_t* aff_class;   /* [n_pods] row of the affinity bit table (bs_upload_affinity) the pod must
                                  match besides sel_mask, or BS_AFF_NONE; the column may be NULL (all NONE)  */
} bs_pod_table;

/* Group table: PGStatusCache.PGStatusMap flattened (cache.go:45-67); canonical
 * iteration order = table index (the reference iterates a Go map, core.go:703). */
typedef struct {
  uint32_t n_groups;
  uint32_t n_lanes;
  const uint32_t* min_member;      /* Spec.MinMember                  types.go:83  */
  const uint32_t* scheduled;       /* Status.Scheduled                types.go:114 */
  const uint32_t* matched;         /* len(MatchedPodNodes.Items()) carried in      */
  const uint8_t* flags;            /* BS_GROUP_*                                   */
  const int64_t* min_res;          /* [n_lanes][n_groups] Spec.MinResources as a Resource */
  const uint32_t* min_res_present; /* scalar keys present in MinResources          */
  const uint64_t* rep_sel;         /* selector mask of pgs.Pod (first-seen pod)    */
  const uint64_t* rep_tol;         /* toleration mask of pgs.Pod                   */
  const int64_t* creation_ns;      /* PodGroup CreationTimestamp      core.go:400  */
  const uint32_t* name_rank;       /* rank of the bare pgName, byte-wise ascending; equal names share a rank (core.go:404) */
  const uint32_t* rep_aff_class;   /* affinity class of pgs.Pod, or BS_AFF_NONE; the column may be NULL     */
} bs_group_table;

/* What one evaluation materialises in HBM besides the decision vectors. */
#define BS_OUT_FIT_BITMAP 0x1u /* P x ceil(N/32) u32 words, bit n%32 of word n/32 */
#define BS_OUT_SCORE 0x2u      /* P x N int64 residual-capacity scores            */
#define BS_OUT_FILTER 0x4u     /* P x ceil(N/32) u32: Filter verdict bit per (pod,node) — ScheduleOperation.Filter /
                                  computeResourceSatisfied (core.go:170-191, 514-564) against the round's max group */
#define BS_OUT_TOPK 0x8u       /* P x K: each pod's K best fitting nodes and their scores (bs_fetch_topk_rows),
                                  without the score matrix; not combinable with BS_OUT_SCORE */
#define BS_TOPK_MAX 32         /* largest list length K */
#define BS_OUT_REASONS 0x10u   /* P x (4 + n_lanes) u32: per pod, how many nodes reject it for each reason
                                  (bs_fetch_reason_rows); combines with every other flag */
#define BS_OUT_PRIORITY 0x20u  /* P x K: each pod's K best fitting nodes under kube-scheduler's resource priorities
                                  (bs_fetch_priority_rows); combines with every other flag, K = bs_config.topk */

/* Bins of a reason row.  A node counts in no bin <=> the pod fits it (fit bitmap bit set); a guarded node counts in
 * exactly one of bins 0-1 (precedence nil, Node()==nil, unschedulable, Taints() error, core.go:606-617,639); a node
 * passing the guards may count in both bins 2 and 3 (checkFit appends both predicates' reasons, core.go:741-759);
 * only a node passing the guards and checkFit counts in lane bins, in every lane that is short
 * (compareResourceAndRequire's rules at percent 1.0, core.go:672-699, without its early return). */
#define BS_REASON_UNSCHEDULABLE 0 /* Spec.Unschedulable (and not nil / no Node())          */
#define BS_REASON_UNAVAILABLE 1   /* nil info, nil Node(), or Taints() returned an error    */
#define BS_REASON_SELECTOR 2      /* node selector / required node affinity not matched     */
#define BS_REASON_TAINTS 3        /* a NoSchedule / NoExecute taint not tolerated           */
#define BS_REASON_LANE0 4         /* + d: resource lane d short ("Insufficient <resource>") */

typedef struct {
  int32_t device;      /* CUDA device ordinal */
  uint32_t n_lanes;    /* lanes of every table uploaded to this engine */
  uint32_t out_flags;  /* BS_OUT_* */
  uint32_t topk;       /* list length K: 1..BS_TOPK_MAX with BS_OUT_TOPK or BS_OUT_PRIORITY, 0 without either (else
                          bs_create -> BS_E_INVAL); with both flags both lists have length K */
} bs_config;

/* Host result buffers; any pointer may be NULL (that output is not copied back). */
typedef struct {
  uint8_t* prefilter;       /* [P] bs_prefilter_code                            */
  uint32_t* feasible_count; /* [P] number of nodes the pod fits on              */
  int32_t* best_node;       /* [P] argmax residual score (lowest index on ties), -1 if none */
  int64_t* best_score;      /* [P] its score, INT64_MIN if none                 */
  uint8_t* admit;           /* [G] bs_admit_code                                */
  uint32_t* admit_bitmap;   /* [ceil(G/32)] bit g set <=> admit[g]==BS_ADMIT    */
  uint8_t* new_denied;      /* [G] 1 if a pod of g hit "cluster resource not enough" (core.go:142,163) */
  uint32_t* order;          /* [P] queue order: pod indices sorted by Less      */
  uint32_t* rank;           /* [P] dense rank of each pod under Less (equal keys share a rank) */
  int32_t max_group;        /* out: findMaxPG winner, -1 if none (core.go:701)  */
  uint32_t max_finished;    /* out: its progress value                          */
  uint8_t* filter_code;     /* [P] bs_filter_code when it does not depend on the node (BS_OUT_FILTER) */
} bs_results;

typedef struct {
  int32_t code;         /* bs_code */
  int32_t reason;       /* bs_prefilter_code */
  int32_t group;        /* group index the message refers to, or -1 */
} bs_status;

typedef struct {
  int32_t ready;        /* core.Permit's first return value (core.go:303-307) */
  int32_t code;         /* bs_code after the adapter mapping (batchscheduler.go:183-201) */
  int64_t wait_ns;      /* waitTime+1s, 0 for Success, DefaultWaitTime for Unschedulable */
  int32_t start_signal; /* 1 when the adapter would fire sendStartScheduleSignal (:197-199) */
  int32_t group;
} bs_permit_result;

/* ---- lifecycle.  Replaces batch.New / core.NewScheduleOperation
 *      (batchscheduler.go:377, core.go:64-77). ---- */
int bs_abi_version(void);
int bs_create(const bs_config* cfg, bs_engine** out);
void bs_destroy(bs_engine* e);
const char* bs_strerror(int err);
const char* bs_last_error(const bs_engine* e);

/* ---- snapshot upload.  Replaces the reads of
 *      frameworkHandler.SnapshotSharedLister().NodeInfos().List() (core.go:597),
 *      PGStatusCache.PGStatusMap (cache.go:45-49) and the per-pod inputs of
 *      PreFilter/Permit/Compare (core.go:88,268,368).  Host arrays are copied;
 *      nothing is retained.  The copy runs under the validation pass: a table
 *      that fails it (BS_E_RANGE) is dropped, and the engine answers BS_E_STATE
 *      until a valid table of that kind is uploaded. ---- */
int bs_upload_nodes(bs_engine* e, const bs_node_table* t);
/* Incremental snapshot update: overwrite rows idx[0..t->n_nodes) of the uploaded node table with
 * the rows of `t` (a compact table of the changed nodes, same lane layout).  The snapshot's list
 * order and size do not change; between scheduling cycles only a few NodeInfos differ. */
int bs_update_nodes(bs_engine* e, const uint32_t* idx, const bs_node_table* t);
int bs_upload_groups(bs_engine* e, const bs_group_table* t);
/* The same for PodGroup state: overwrite rows idx[0..t->n_groups) of the uploaded group table.
 * Between cycles a few groups change (matched count, Status.Scheduled, the Scheduled / denied flags,
 * MinResources and the representative pod once the first pod arrived: cache.go:52-67); the table's
 * size and order stay. */
int bs_update_groups(bs_engine* e, const uint32_t* idx, const bs_group_table* t);
int bs_upload_pods(bs_engine* e, const bs_pod_table* t);
/* checkFit beyond bit masks (core.go:741-759 -> predicates.PodMatchNodeSelector).  sel_mask / label_mask
 * carry nodeSelector pairs exactly (<= 64 distinct pairs per round); REQUIRED node-affinity terms
 * (matchExpressions with In / NotIn / Exists / DoesNotExist / Gt / Lt, matchFields, ORed terms) and any
 * overflow of the 64 pairs travel as an explicit table: the caller groups pods into affinity classes,
 * evaluates each class against every node of the uploaded snapshot and uploads
 *     bits[n_classes][ceil(n_nodes / 32)]   bit n%32 of word n/32 of row c = class c matches node n.
 * A pod fits a node iff the mask test AND its class's bit hold (bs_pod_table.aff_class, BS_AFF_NONE =
 * mask test only); the group's representative pod likewise (bs_group_table.rep_aff_class).  The table
 * belongs to the node snapshot: bs_upload_nodes drops it (upload nodes, then the table), n_classes = 0
 * clears it.  A class id >= n_classes at evaluation time is BS_E_INDEX. */
int bs_upload_affinity(bs_engine* e, uint32_t n_classes, const uint32_t* bits);
/* max_schedule_time: plugin arg (batchscheduler.go:71-75, util.GetWaitTimeDuration
 * k8s.go:82-91).  per_group_ns may be NULL; entries < 0 mean "unset". */
int bs_set_wait_time(bs_engine* e, int64_t default_ns, const int64_t* per_group_ns,
                     uint32_t n_groups);

/* ---- one round over the uploaded snapshot.  Replaces, batched over every pod
 *      of the round: ScheduleOperation.PreFilter (core.go:88-167) incl. findMaxPG
 *      (:701-739), getPreAllocatedResource (:774-793), compareClusterResourceAndRequire
 *      (:595-632), singleNodeResource (:634-670), compareResourceAndRequire
 *      (:672-699); the Permit readiness count (core.go:303); Compare (core.go:368-411).
 *      bs_evaluate = bs_evaluate_async + bs_fetch. ---- */
int bs_evaluate(bs_engine* e, bs_results* out);
int bs_evaluate_async(bs_engine* e);       /* enqueue the kernels, no host sync */
int bs_sync(bs_engine* e);                 /* wait for the engine stream        */
int bs_fetch(bs_engine* e, bs_results* out);
/* bs_fetch without the copy: waits for the round, brings every decision vector to the host in one DMA and POINTS the
 * array fields of *out into the engine's pinned decision arena (filter_code: null without BS_OUT_FILTER).  The
 * pointers and their contents stay valid until the next bs_evaluate* / bs_upload_* / bs_update_* / bs_destroy on
 * this engine; the caller must not write through them.  (A scheduler reads the verdicts once per cycle: copying
 * 2.6 MB out of the arena costs as much as the DMA that filled it.) */
int bs_evaluate_view(bs_engine* e, bs_results* out);
int bs_fetch_view(bs_engine* e, bs_results* out);

/* ---- per-call mirrors answering from the last evaluation ---- */
/* batchSchedulingPlugin.PreFilter  (batchscheduler.go:102-108) */
int bs_prefilter(bs_engine* e, uint32_t pod, bs_status* st);
/* batchSchedulingPlugin.Permit     (batchscheduler.go:165-202) */
int bs_permit(bs_engine* e, uint32_t pod, uint32_t node, bs_permit_result* r);
/* batchSchedulingPlugin.Less       (batchscheduler.go:214-216); returns 1/0 or <0 */
int bs_less(bs_engine* e, uint32_t pod_a, uint32_t pod_b);
/* batchSchedulingPlugin.Filter (batchscheduler.go:151-157) -> core.Filter (core.go:170-191).  Needs
 * BS_OUT_FILTER.  st->reason is a bs_filter_code; code Success / Unschedulable. */
int bs_filter(bs_engine* e, uint32_t pod, uint32_t node, bs_status* st);
/* Formats the reference's error string for a status (core.go:102,107,143,505,509).
 * ns_name is the "namespace/name" of the group, occupied_by the OccupiedBy text. */
int bs_format_message(const bs_status* st, const char* ns_name, const char* occupied_by,
                      char* buf, size_t buf_len);

/* ---- gang state: the TTL tables around Permit as ENGINE state (SURVEY.md 8(f) row 3) ----
 * The reference keeps, per PodGroup, MatchedPodNodes (uid -> pod/node pair) and PodNameUIDs ("ns/name" -> uid),
 * both go-cache maps with a per-entry TTL of the group's wait time (controller.go:314-335, core.go:283-300), plus
 * the scheduler-wide lastDeniedPG (20 s) and lastPermittedPod (2 s) caches (core.go:71-72,188,423-425).  These
 * calls keep them inside the engine, driven by the caller's clock (now_ns); uids and pod names cross the ABI as
 * 64-bit ids (the Go shim hashes the strings).
 *   bs_state_reset    empty tables for the uploaded group table
 *   bs_state_remap    carry the tables over to a group table of another shape
 *   bs_set_pod_ids    uid and "ns/name" id of every pod of the uploaded pod table
 *   bs_begin_cycle    writes the tables' view at now_ns into the round's inputs — matched[g] =
 *                     len(MatchedPodNodes.Items()), the SCHEDULED (pgs.Scheduled) and DENIED flags, the pods'
 *                     PERMITTED_RECENTLY flag — replacing those columns of the uploaded tables; after the round,
 *                     every group with new_denied set is added to the deny table (core.go:142,163)
 *   bs_permit_at      ScheduleOperation.Permit with its bookkeeping (core.go:268-309): Set / Delete-old-uid / Set,
 *                     ready = uint32(len(Items())) >= MinMember - Status.Scheduled, pgs.Scheduled on ready; the
 *                     adapter mapping of bs_permit (batchscheduler.go:165-202)
 *   bs_expire         one janitor tick: a group whose PodNameUIDs holds an expired entry rejects every matched
 *                     pod ("Group failed", batchscheduler.go:347-354), forgets them, flushes its names and is
 *                     deny-listed for 20 s (controller.go:322-333); returns the (group, uid) pairs to reject
 *                     and the evicted groups (counts may exceed the capacities: call again with larger buffers
 *                     is NOT possible, size them for the worst case = pods in flight)
 *   bs_allow_list     StartBatchSchedule's Allow loop (batchscheduler.go:292-344): the uids (and the nodes they
 *                     were permitted on) to Allow when the group has enough waiting pods, removed from the table
 *   bs_deny / bs_mark_permitted   AddToDenyCache (core.go:423) / lastPermittedPod.Add (core.go:188)
 *   bs_group_state    read-back for tests and metrics */
int bs_state_reset(bs_engine* e);
/* the group table is about to change shape (PodGroups created / deleted): row g of the NEXT table continues
 * row old_index[g] of the current one (-1: a new group, empty tables); call before bs_begin_cycle */
int bs_state_remap(bs_engine* e, uint32_t n_groups, const int32_t* old_index);
/* bulk read-backs for a packer that needs the flags before it builds the round's tables: per group
 * len(MatchedPodNodes.Items()) and BS_GROUP_SCHEDULED | BS_GROUP_DENIED; per uid lastPermittedPod membership */
int bs_state_view(bs_engine* e, int64_t now_ns, uint32_t n_groups, uint32_t* matched, uint8_t* flags);
int bs_permitted_view(bs_engine* e, int64_t now_ns, const uint64_t* uids, uint32_t n, uint8_t* out);
/* hands the tables of `src` over to `dst` (an engine re-created with another lane count keeps its history) */
int bs_state_move(bs_engine* dst, bs_engine* src);
int bs_set_pod_ids(bs_engine* e, const uint64_t* uid /* [n_pods] */, const uint64_t* name_id /* [n_pods] */);
int bs_begin_cycle(bs_engine* e, int64_t now_ns);
int bs_permit_at(bs_engine* e, uint32_t pod, uint32_t node, int64_t now_ns, bs_permit_result* r);
int bs_expire(bs_engine* e, int64_t now_ns, uint32_t* rej_group, uint64_t* rej_uid, uint32_t rej_cap, uint32_t* n_rejected,
              uint32_t* evicted_group, uint32_t evict_cap, uint32_t* n_evicted);
int bs_allow_list(bs_engine* e, uint32_t group, int64_t now_ns, uint64_t* uids, uint32_t* nodes, uint32_t cap, uint32_t* n);
int bs_deny(bs_engine* e, uint32_t group, int64_t now_ns);
int bs_mark_permitted(bs_engine* e, uint64_t uid, int64_t now_ns);
int bs_group_state(bs_engine* e, uint32_t group, int64_t now_ns, uint32_t* matched, int32_t* scheduled_flag, int32_t* denied);

/* ---- standalone table kernels (unit-level parity with the reference helpers) ---- */
/* singleNodeResource over every node for one (sel,tol) pod class and percent
 * (core.go:634-670).  left: [n_lanes][n_nodes], present: [n_nodes]. */
int bs_node_left(bs_engine* e, uint64_t sel, uint64_t tol, float percent,
                 int64_t* left, uint32_t* present);
/* compareClusterResourceAndRequire for explicit needs (core.go:595-632):
 * n_needs need vectors [n_lanes][n_needs] + presence masks -> ok[n_needs]. */
int bs_cluster_check(bs_engine* e, uint64_t sel, uint64_t tol, float percent,
                     const int64_t* need, const uint32_t* need_present, uint32_t n_needs,
                     uint8_t* ok);

/* ---- multi-round admission on the device (SURVEY.md 8(f) row 4) ----
 * The reference schedules one pod per cycle against MUTABLE state: PreFilter reads the live group
 * cache and snapshot (core.go:88-167), the chosen node's `requested` grows when the pod is assumed
 * (NodeInfo.AddPod), Permit records the match and may mark the group Scheduled (core.go:268-309), a
 * failed cluster check freezes the group (AddToDenyCache, core.go:423-425).  bs_replay walks `queue`
 * (pod indices in pop order; NULL = table order, n_queue = number of pods) through exactly that
 * cycle in ONE kernel, starting from the uploaded tables, which stay untouched.  The node a passing
 * pod is assumed onto is the first node in list order where it fits (the stand-in for the upstream
 * Filter/Score/selectHost the repo's oracle uses as well).  Sequential by nature: one GPU, no
 * sharding ("replicas only").
 * Outputs per queue position; the optional after-state arrays (NULL = not wanted) return the
 * mutated copies so that the caller can continue from them (bs_upload_* / bs_update_nodes).
 * bs_replay_priority (below, after the resource priorities) is the same walk with kube-scheduler's
 * node choice in place of first-fit. */
typedef struct bs_replay_result {
  uint8_t* prefilter;          /* [n_queue] bs_prefilter_code */
  int32_t* node;               /* [n_queue] assumed node, -1 none */
  uint8_t* ready;              /* [n_queue] Permit returned ready (core.go:303) */
  int64_t* node_requested;     /* [n_lanes][n_nodes] or NULL */
  int32_t* node_pod_count;     /* [n_nodes] or NULL */
  uint32_t* node_req_present;  /* [n_nodes] or NULL; an assumed pod adds its keys of lanes 4..n_lanes-1 only */
  uint32_t* group_matched;     /* [n_groups] or NULL */
  uint8_t* group_flags;        /* [n_groups] or NULL (BS_GROUP_*) */
  int64_t* group_min_res;      /* [n_lanes][n_groups] or NULL */
  uint32_t* group_min_res_present; /* [n_groups] or NULL; a group's first pod gives its whole mask, bits 0..3 cleared */
  uint64_t* group_rep_sel;     /* [n_groups] or NULL */
  uint64_t* group_rep_tol;     /* [n_groups] or NULL */
} bs_replay_result;
int bs_replay(bs_engine* e, const uint32_t* queue, uint32_t n_queue, bs_replay_result* out);

/* ---- device-side access for callers that keep results in HBM (bench, NCCL) ---- */
typedef enum {
  BS_BUF_FIT_BITMAP = 0,
  BS_BUF_SCORE = 1,
  BS_BUF_ADMIT_BITMAP = 2,
  BS_BUF_PREFILTER = 3,
  BS_BUF_ADMIT = 4,
  BS_BUF_ORDER = 5,
  BS_BUF_GATHERED_ADMIT = 6
} bs_buffer;
int bs_device_buffer(bs_engine* e, int which, void** dev_ptr, size_t* bytes);
void* bs_stream(bs_engine* e); /* the cudaStream_t a round is ordered on: uploads, the fit kernel and the
                                  verdicts run on it, and the two side streams of a round (PreFilter chain,
                                  queue sort) join it before the round ends, so work enqueued on it after
                                  bs_evaluate_async sees every result */
/* elements per row of the score matrix in HBM (BS_BUF_SCORE): n_nodes rounded up to even, so that every
 * row starts on a 16-byte boundary (the kernel writes row segments with TMA bulk stores); the pad
 * element of an odd-sized table holds no score.  bs_fetch_score_rows returns dense [n][n_nodes] rows. */
uint32_t bs_score_pitch(const bs_engine* e);
/* words per row of the fit bitmap in HBM (BS_BUF_FIT_BITMAP): ceil(n_nodes / 32) rounded up to 32, so that every
 * row is a whole number of 128-byte lines (the kernel writes one aligned line per pod and 1024 nodes);
 * bs_fetch_fit_rows returns dense [n][ceil(n_nodes / 32)] rows. */
uint32_t bs_bitmap_pitch(const bs_engine* e);
/* copy rows [pod0, pod0+n) of the fit bitmap / score matrix to the host */
int bs_fetch_fit_rows(bs_engine* e, uint32_t pod0, uint32_t n, uint32_t* words);
int bs_fetch_score_rows(bs_engine* e, uint32_t pod0, uint32_t n, int64_t* scores);
int bs_fetch_filter_rows(bs_engine* e, uint32_t pod0, uint32_t n, uint32_t* words);
/* copy the top-K lists of pods [pod0, pod0+n) to the host as dense [n][K] rows (BS_OUT_TOPK).  Row p holds the
 * fitting nodes of pod p ordered by score descending, then node index ascending (entry 0 = best_node / best_score),
 * min(K, feasible_count[p]) of them, padded with node -1 and score INT64_MIN.  Either pointer may be NULL. */
int bs_fetch_topk_rows(bs_engine* e, uint32_t pod0, uint32_t n, int32_t* nodes, int64_t* scores);
/* copy the reason rows of pods [pod0, pod0+n) to the host as dense [n][4 + n_lanes] counters (BS_OUT_REASONS): bin b
 * of row p = the number of snapshot nodes that reject pod p for reason b (BS_REASON_*) */
int bs_fetch_reason_rows(bs_engine* e, uint32_t pod0, uint32_t n, uint32_t* counts);
/* kube-scheduler's FailedScheduling text for one reason row (no engine, no device):
 *     "0/<n_nodes> nodes are available: <count> <reason>, ... ."
 * one entry per non-zero bin, entries sorted as whole strings byte-wise ascending (Go's sort.Strings), joined by
 * ", ".  Lane d >= 4 reads "Insufficient <scalar_names[d - 4]>", or "Insufficient lane<d>" when scalar_names is NULL.
 * A buffer too small for the whole message is BS_E_INVAL (nothing is truncated). */
int bs_format_fit_error(const uint32_t* counts, uint32_t n_lanes, uint32_t n_nodes, const char* const* scalar_names,
                        char* buf, size_t buf_len);

/* ---- resource priorities (BS_OUT_PRIORITY): kube-scheduler v1.17's NodeResourcesLeastAllocated,
 *      NodeResourcesMostAllocated and NodeResourcesBalancedAllocation over each pod's fitting nodes ----
 * For pod p and node n, with cap = alloc[0..1][n] (unscaled) and req = node_nz[n] + pod_nz[p] per resource:
 *     least(r, c) = c == 0 || r > c ? 0 : (c - r) * 100 / c      most(r, c) = c == 0 || r > c ? 0 : r * 100 / c
 *     Least = (least(cpu) + least(mem)) / 2        Most = (most(cpu) + most(mem)) / 2        (int64, truncating)
 *     frac(r, c) = c == 0 ? 1.0 : (double)r / (double)c                      (IEEE binary64, round to nearest)
 *     Balanced = fc >= 1 || fm >= 1 ? 0 : (int64)((1.0 - fabs(fc - fm)) * 100.0)   (toward zero; below -2^63:
 *                INT64_MIN)
 *     score = w_least * Least + w_most * Most + w_balanced * Balanced        (int64, two's complement wrap)
 * Only the pod's fitting nodes are scored (fit bitmap bit set).  The non-zero columns are caller-supplied: per pod
 * the sum over its containers of the Requests with an absent cpu key counted as 100 (millicores) and an absent memory
 * key as 209715200 (bytes; an explicit zero stays zero); per node the same sum over the pods on it
 * (NodeInfo.NonZeroRequest()).  Values lie in [0, BS_NONZERO_MAX]. */
#define BS_NONZERO_MAX (1ll << 56)
/* weights of the three scores (default 1, 0, 1: v1.17's default provider); any time, read by the next evaluation */
int bs_set_score_weights(bs_engine* e, uint32_t least, uint32_t most, uint32_t balanced);
/* nz[2][n_nodes]: row 0 cpu (millicores), row 1 memory (bytes).  n_nodes must equal the uploaded node table's
 * (else BS_E_INVAL); a value outside [0, BS_NONZERO_MAX] is BS_E_RANGE and drops the column.  The column belongs to the
 * node snapshot: bs_upload_nodes and bs_update_nodes drop it. */
int bs_upload_node_nonzero(bs_engine* e, uint32_t n_nodes, const int64_t* nz);
/* nz[2][n_pods], the same for the pod table; bs_upload_pods drops it.  An evaluation with BS_OUT_PRIORITY and either
 * column missing is BS_E_STATE before anything is launched. */
int bs_upload_pod_nonzero(bs_engine* e, uint32_t n_pods, const int64_t* nz);
/* copy the priority lists of pods [pod0, pod0+n) to the host as dense [n][K] rows (BS_OUT_PRIORITY).  Row p holds
 * the fitting nodes of pod p ordered by score descending, then node index ascending, min(K, feasible_count[p]) of
 * them, padded with node -1 and score INT64_MIN.  Either pointer may be NULL. */
int bs_fetch_priority_rows(bs_engine* e, uint32_t pod0, uint32_t n, int32_t* nodes, int64_t* scores);
/* bs_replay with kube-scheduler's node choice: the same walk (PreFilter on live state, fillOccupiedObj, findMaxPG, the
 * cluster scans, assume, Permit, the after-state), except that a passing pod goes to the node with the highest score
 * above among the nodes where it fits on the live state (visited, Taints() ok, checkFit of its own class, every lane
 * at percent 1.0), ties to the lower node index, -1 when none fits: entry 0 of a BS_OUT_PRIORITY list computed on the
 * live state, with the weights of bs_set_score_weights.  Assume debits `requested` by the pod table's request as
 * bs_replay does and adds the pod's non-zero column to the chosen node's live one; node_nonzero_after ([2][n_nodes] or
 * NULL) returns that column.  Both non-zero columns must be uploaded (else BS_E_STATE before anything is launched;
 * BS_OUT_PRIORITY at bs_create is not needed); they stay untouched.  BS_E_RANGE when, for either row, the column
 * maxima give max(node) + n_queue * max(pod) > 2^62.  Timed under BS_K_REPLAY. */
int bs_replay_priority(bs_engine* e, const uint32_t* queue, uint32_t n_queue, bs_replay_result* out,
                       int64_t* node_nonzero_after);
/* kube-scheduler v1.17's RequestedToCapacityRatio priority, added to the BS_OUT_PRIORITY score with weight `weight`
 * (0 = off, the default).  Shape: n_points (1..101) points, utilization strictly ascending in [0, 100], score in
 * [0, 100] (node-score units).  lane_weight[n_lanes] (n_lanes = the engine's), lane 3 must be 0; absent_weight = the
 * weights of resources with capacity 0 on every node.  Sum of lane weights + absent_weight <= 2^24.  Else BS_E_INVAL,
 * and the previous setting stays.  Read by the next evaluation and by bs_replay_priority.
 * Per (pod p, node n) and weighted lane d [upstream, from memory]:
 *     c = alloc[d][n] (unscaled); r = node_nz[n] + pod_nz[p] on lanes 0-1, requested[d][n] + req[d][p] on lane 2 and
 *         the scalar lanes, a scalar key absent on a side counting 0 there (alloc_present / req_present); the pod side
 *         is the pod table's request (Limits else Requests), which for extended resources and hugepages equals
 *         Requests
 *     util = c == 0 || r > c ? 100 : 100 - (c - r) * 100 / c     (int64, wrapping, truncating toward zero)
 *     s_d = shape(util): s_0 at or below u_0, s_last above the last point, else on the segment u_{i-1} < util <= u_i
 *           s_{i-1} + (s_i - s_{i-1}) * (util - u_{i-1}) / (u_i - u_{i-1})  (int64, truncating toward zero)
 *     Ratio = round(sum s_d * w_d / sum w_d) over the resources with s_d > 0 (half away from zero; 0 without any);
 *             absent_weight joins both sums with s = shape(100) when shape(100) > 0
 *     score = w_least * Least + w_most * Most + w_balanced * Balanced + weight * Ratio   (int64, two's complement wrap)
 * v1.17's policy file gives shape scores in 0..10 and the scheduler multiplies them by 10: the caller scales. */
int bs_set_ratio_priority(bs_engine* e, uint32_t weight, uint32_t n_points, const uint32_t* utilization,
                          const uint32_t* score, uint32_t n_lanes, const uint32_t* lane_weight, uint32_t absent_weight);
/* kube-scheduler v1.17's TaintToleration and (preferred) NodeAffinity priorities, added to the BS_OUT_PRIORITY score
 * with weights taint_toleration and node_affinity (0, 0 = off, the default; v1.17's default profile is 1, 1).  Any
 * time, read by the next evaluation.  Per (pod p, node n) [upstream, from memory]:
 *     t(p, n) = popcount(prefer_taints[n] & ~prefer_tol[p])   the node's PreferNoSchedule taints p does not tolerate
 *     a(p, n) = pref_weights[pref_class[p]][n], 0 for BS_PREF_NONE   the weights of p's preferred terms n matches
 *     Mt, Ma = the maxima of t and a over the pod's fit set (the nodes of its fit-bitmap row; no other node counts)
 *     TT = Mt == 0 ? 100 : 100 - 100 * t / Mt         NA = Ma == 0 ? 0 : 100 * a / Ma       (int64, truncating)
 *     score = <the score above> + taint_toleration * TT + node_affinity * NA                 (int64, two's complement wrap)
 * An evaluation with BS_OUT_PRIORITY and a non-zero weight is BS_E_STATE before anything is launched when a column it
 * needs is missing (taint_toleration: both masks; node_affinity: the weight table and the class column), and
 * BS_E_INDEX when node_affinity is non-zero and a pod's class is >= n_classes.  bs_replay_priority refuses to run
 * (BS_E_INVAL) while either weight is non-zero. */
int bs_set_node_priority_weights(bs_engine* e, uint32_t taint_toleration, uint32_t node_affinity);
#define BS_PREF_NONE 0xffffffffu                 /* pref_class of a pod without preferred terms (a = 0) */
#define BS_PREF_TABLE_MAX_BYTES (1ull << 30)     /* n_classes x Npad x 4 (Npad: n_nodes rounded up) at most 1 GiB */
/* prefer_taints[n_nodes]: bit b = the node carries the round's PreferNoSchedule taint b (the caller's dictionary of
 * distinct key/value pairs, at most 64); pref_weights[n_classes][n_nodes]: a(class, node), each in [0, INT32_MAX].
 * n_nodes must equal the node table's (else BS_E_INVAL), a table above BS_PREF_TABLE_MAX_BYTES is BS_E_INVAL, a
 * negative weight BS_E_RANGE; a failing call leaves the side dropped.  The side belongs to the node snapshot:
 * bs_upload_nodes and bs_update_nodes drop it. */
int bs_upload_node_preferences(bs_engine* e, uint32_t n_nodes, const uint64_t* prefer_taints, uint32_t n_classes,
                               const int32_t* pref_weights);
/* prefer_tol[n_pods]: the bits of the dictionary each pod tolerates; pref_class[n_pods]: its row of pref_weights or
 * BS_PREF_NONE.  n_pods must equal the pod table's (else BS_E_INVAL); bs_upload_pods drops the side. */
int bs_upload_pod_preferences(bs_engine* e, uint32_t n_pods, const uint64_t* prefer_tol, const uint32_t* pref_class);
/* kube-scheduler v1.17's ImageLocality and NodePreferAvoidPods priorities, added to the BS_OUT_PRIORITY score and to
 * bs_replay_priority's node choice with weights image_locality and prefer_avoid_pods (0, 0 = off, the default;
 * v1.17's default profile is 1, 10000).  Any time, read by the next evaluation and by bs_replay_priority.  Both terms
 * are static per (pod, node): nothing is normalized over the fit set.  Per (pod p, node n) [upstream, from memory]:
 *     NumNodes(i) = the snapshot nodes whose bit of name i is set (every node of the table counts, fitting or not)
 *     scaled(i) = (int64)((double)image_size[i] * ((double)NumNodes(i) / (double)n_nodes))
 *                 (binary64, round to nearest, then truncation toward zero)
 *     sum = the sum of scaled(i) over the ids i of p's class (a repeated id counts again) whose bit is set on n
 *     IL = 100 * (clamp(sum, 23 MiB, 1000 MiB) - 23 MiB) / 977 MiB       (int64, truncating; 0 for BS_IMAGE_NONE)
 *     NPA = avoid_bit[p] != BS_AVOID_NONE && bit avoid_bit[p] of avoid_mask[n] is set ? 0 : 100
 *     score = <the score above> + image_locality * IL + prefer_avoid_pods * NPA   (int64, two's complement wrap)
 * The caller builds the image dictionary from the names the nodes report (Status.Images[].Names, as reported) that
 * some pod's normalized container image matches (":latest" appended when the last ':' is not after the last '/'); only
 * Spec.Containers count.  Builder-defined: NumNodes is counted over the current snapshot, and a name reported with
 * different sizes takes the size of the lowest node index that reports it.  avoid_bit is the pod's controller of kind
 * ReplicationController or ReplicaSet in the caller's controller dictionary (at most 64); the caller parses the nodes'
 * preferAvoidPods annotations, one that fails to parse listing nothing.
 * An evaluation with BS_OUT_PRIORITY, or bs_replay_priority, with a non-zero weight is BS_E_STATE before anything is
 * launched when a column it needs is missing (image_locality: the bit rows and sizes, and the pod classes;
 * prefer_avoid_pods: the avoid masks and the pod bits), and BS_E_INDEX when image_locality is non-zero and a pod's
 * class is >= n_classes or a class lists an id >= n_images, and BS_E_INVAL when image_locality is non-zero and
 * n_classes x Npad passes BS_LOC_TABLE_MAX_BYTES for the node table of now.  The class x node IL table is rebuilt on the device at the
 * first evaluation (or walk) after either side or a weight changes. */
int bs_set_locality_weights(bs_engine* e, uint32_t image_locality, uint32_t prefer_avoid_pods);
#define BS_IMAGE_NONE 0xffffffffu                /* image_class of a pod without dictionary images (IL = 0) */
#define BS_AVOID_NONE 0xffu                      /* avoid_bit of a pod without an RC / RS controller (NPA = 100) */
#define BS_IMAGE_SIZE_MAX (1ll << 48)            /* largest image size, in bytes */
#define BS_LOC_CLASS_MAX 64                      /* ids one image class may list: every sum stays below 2^54 */
#define BS_LOC_TABLE_MAX_BYTES (1ull << 30)      /* n_images x ceil(n_nodes/32) x 4, and n_classes x Npad, each <= 1 GiB */
/* image_size[n_images]: bytes, each in [0, BS_IMAGE_SIZE_MAX] (else BS_E_RANGE); image_bits[n_images][ceil(n_nodes/32)]:
 * bit n%32 of word n/32 of row i = node n reports name i; avoid_mask[n_nodes]: bit b = the node's preferAvoidPods
 * annotation lists controller b of the round's dictionary.  image_size and image_bits may be NULL while image_locality
 * is 0, avoid_mask while prefer_avoid_pods is 0 (the side then lacks that part).  n_nodes must equal the node table's
 * (else BS_E_INVAL), a bit table above BS_LOC_TABLE_MAX_BYTES is BS_E_INVAL; a failing call leaves the side dropped.
 * The side belongs to the node snapshot: bs_upload_nodes and bs_update_nodes drop it. */
int bs_upload_node_locality(bs_engine* e, uint32_t n_nodes, uint32_t n_images, const int64_t* image_size,
                            const uint32_t* image_bits, const uint64_t* avoid_mask);
/* image_class[n_pods]: the pod's class or BS_IMAGE_NONE; class_offset[n_classes + 1] (ascending from 0) and
 * class_images[class_offset[n_classes]]: the dictionary ids of each class, at most BS_LOC_CLASS_MAX per class (else
 * BS_E_INVAL); avoid_bit[n_pods]: 0..63 or BS_AVOID_NONE (else BS_E_RANGE).  image_class, class_offset and
 * class_images may be NULL while image_locality is 0, avoid_bit while prefer_avoid_pods is 0.  n_pods must equal the
 * pod table's, n_classes x Npad bytes may not pass BS_LOC_TABLE_MAX_BYTES (else BS_E_INVAL); a failing call leaves the
 * side dropped.  bs_upload_pods drops the side. */
int bs_upload_pod_locality(bs_engine* e, uint32_t n_pods, const uint32_t* image_class, uint32_t n_classes,
                           const uint32_t* class_offset, const uint32_t* class_images, const uint8_t* avoid_bit);

/* ---- preemption: PreFilterExtensions.RemovePod and the node / victims kube-scheduler's preemption would pick ----
 * The bound-pod table lists the pods already running on the snapshot's nodes (NodeInfo.Pods()).  Rows may come in
 * any order; the engine groups them by node in MoreImportantPod order (priority descending, start time ascending,
 * then table index ascending).  Validation: node >= n_nodes or gid < BS_GID_MISSING is BS_E_INDEX; more rows on a node than its pod_count,
 * or scalar keys that are not a subset of the node's req_present, BS_E_INVAL; a value or any per-node suffix sum of
 * a lane beyond +-BS_VALUE_LIMIT, BS_E_RANGE.  A failing table is dropped.  The table belongs to the node snapshot:
 * bs_upload_nodes, bs_update_nodes and bs_upload_groups drop it (BS_E_STATE until it is uploaded again). */
#define BS_BOUND_GROUP_LOCKED 0x01u /* the pod's PodGroup Status.Phase is Scheduled or Running (core.go:235-236) */
typedef struct {
  uint32_t n_pods, n_lanes;
  const uint32_t* node;        /* [V] snapshot index of the node it is bound to (NodeInfo.Pods())              */
  const int64_t* req;          /* [n_lanes][V] what NodeInfo.RemovePod subtracts: the containers' Requests (not
                                  Limits: calculateResource, [upstream, from memory]); lane 3 ignored             */
  const uint32_t* req_present; /* [V] scalar keys; must be a subset of its node's req_present                     */
  const int32_t* gid;          /* [V] group index, BS_GID_NONE (online) or BS_GID_MISSING                          */
  const int32_t* priority;     /* [V] GetPodPriority */
  const int64_t* start_ns;     /* [V] Status.StartTime */
  const uint8_t* flags;        /* [V] BS_BOUND_* */
} bs_bound_table;
int bs_upload_bound_pods(bs_engine* e, const bs_bound_table* t);

/* Result of bs_preempt.  Per preemptor: the node genericScheduler.Preempt -> pickOneNodeForPreemption would pick
 * (-1 none) and, in victims[victim_offset[i] .. victim_offset[i + 1]), the bound-table indices of the pods
 * selectVictimsOnNode would evict there, in reprieve order (most important first). */
typedef struct {
  int32_t* node;            /* [n] chosen node, -1 none                                              */
  uint32_t* n_victims;      /* [n]                                                                   */
  uint32_t* n_candidates;   /* [n] nodes where removing every lower-priority pod lets the pod fit    */
  uint32_t* victim_offset;  /* [n + 1] exclusive scan of n_victims                                   */
  uint32_t* victims;        /* [victims_cap] bound-table indices, per preemptor in reprieve order      */
  uint32_t victims_cap;
  uint32_t victims_total;   /* out, always written; > victims_cap -> BS_E_INVAL, victims untouched   */
} bs_preempt_result;
/* Every pods[i] (an index of the uploaded pod table) is an independent what-if against the uploaded node and bound
 * tables (DESIGN.md §2 "Preemption").  Needs nodes, groups, pods and the bound table; does not depend on, and does not
 * change, any round's state or outputs. */
int bs_preempt(bs_engine* e, const uint32_t* pods, uint32_t n, bs_preempt_result* out);

/* RemovePod verdicts (core.PreemptRemovePod, core.go:203-260) */
typedef enum {
  BS_REMOVE_ALLOW = 0,
  BS_REMOVE_OFFLINE_ONLINE = 1, /* "offline pods %v are forbidden to preempt online %v"                     :217 */
  BS_REMOVE_NOT_FOUND = 2,      /* "can not found pod group: %v"                                            :224 */
  BS_REMOVE_LOCKED = 3,         /* "pod belongs to Scheduled or Running pod group can not be scheduled"     :237 */
  BS_REMOVE_SAME_GROUP = 4      /* "podToSchedule and podToRemove belong to same pod group, do not preempt" :252 */
} bs_remove_code;
/* batchSchedulingPluginExtension.RemovePod (batchscheduler.go:132-144) -> core.PreemptRemovePod (core.go:203-260) for
 * pod `pod` of the pod table and row `bound` of the bound table.  st->reason is a bs_remove_code, st->code Success or
 * Unschedulable, st->group the victim's group or -1.  PreemptAddPod always succeeds (core.go:194-196). */
int bs_remove_pod(bs_engine* e, uint32_t pod, uint32_t bound, bs_status* st);
/* The reference's error text of a RemovePod status ("" for BS_REMOVE_ALLOW); victim_ns_name is "namespace/pgName" of
 * the victim's group.  A buffer too small for the whole message is BS_E_INVAL. */
int bs_format_remove_message(const bs_status* st, const char* pod_name, const char* victim_name,
                             const char* victim_ns_name, char* buf, size_t buf_len);

/* ---- multi-GPU exchange of the admit bitmap over peer memory (NVLink / NVSwitch) ----
 * The path shards over groups (one process per GPU); the only exchange is the all-gather of the
 * per-rank admit bitmaps.  Instead of a separate NCCL launch, bs_evaluate_async ends with a push
 * kernel that writes this rank's bitmap words straight into every peer's gather buffer (CUDA IPC
 * mapped peer memory) and publishes the round number there; a one-warp wait kernel on a side stream
 * waits (bounded) for the peers' words of the same round.  The buffer holds two slot sets (round
 * parity), so the NEXT round's kernels run while the wait is still pending: a late rank stalls its
 * peers only once it is more than one round behind.  No rank ever spins on its main stream.
 *   bs_peer_init    allocate the gather buffer [2][world][words_per_rank] (+ flags) on this GPU
 *   bs_peer_handle  64-byte cudaIpcMemHandle of it, to be exchanged out of band (e.g. torch.distributed)
 *   bs_peer_attach  map every peer's buffer (handles[world][64], own slot ignored)
 *   bs_peer_join    make the engine stream wait for the last round's gathered words (for work the
 *                   caller enqueues on bs_stream; bs_sync and bs_fetch_gathered_admit wait themselves)
 *   bs_fetch_gathered_admit  copy [world][words_per_rank] words of the last round to the host
 * BS_BUF_GATHERED_ADMIT is the device address of the last round's slot set (rank r at word
 * r*words_per_rank); it alternates between two addresses from round to round.
 * Failure: a rank that does not arrive within BS_PEER_TIMEOUT_MS (env, default 2000) makes bs_sync /
 * bs_fetch_gathered_admit return BS_E_PEER; from then on bs_evaluate* fails fast with BS_E_PEER (no
 * further spinning) until every rank has called bs_peer_detach and attached again (a new epoch:
 * buffers zeroed, round numbers restart at 1). */
int bs_peer_init(bs_engine* e, uint32_t rank, uint32_t world, uint32_t words_per_rank);
int bs_peer_handle(bs_engine* e, unsigned char handle[64]);
int bs_peer_attach(bs_engine* e, const unsigned char* handles /* [world][64] */);
int bs_peer_detach(bs_engine* e);
int bs_peer_join(bs_engine* e);
int bs_fetch_gathered_admit(bs_engine* e, uint32_t* words /* [world][words_per_rank] */);

/* ---- measurement hooks ---- */
typedef enum {
  BS_K_NODE_LEFT = 0,
  BS_K_FIND_MAX = 1,
  BS_K_CLASS_PREFIX = 2,
  BS_K_PREFILTER = 3,
  BS_K_GANG_FIT = 4,   /* the dominant kernel: gang_fit_kernel alone (events right around its launch; the tail's memsets and
                          unpack kernel and gang_admit are counted in its launches, not in its time) */
  BS_K_SORT = 5,
  BS_K_FILTER = 6,     /* optional Filter matrix (BS_OUT_FILTER) */
  BS_K_PEER = 7,       /* admit-bitmap exchange over peer memory */
  BS_K_REPLAY = 8,     /* bs_replay: the pod-at-a-time cycle in one persistent kernel */
  BS_K_REASONS = 9,    /* reason rows (BS_OUT_REASONS): the per-pod lane sweep; the per-class bins and gate bitmap are
                          rebuilt with the class fit bits and counted in BS_K_NODE_LEFT */
  BS_K_COUNT = 10
} bs_kernel_id;
int bs_set_profiling(bs_engine* e, int on); /* record CUDA events around each stage */
/* milliseconds of stage k in the last evaluation, and launches it took */
int bs_kernel_ms(bs_engine* e, int k, float* ms, uint32_t* launches);
uint64_t bs_launch_count(const bs_engine* e); /* kernels launched since bs_create */
/* how the last evaluation's fit kernel carried the resource lanes: int64 (wide), int32 (narrow: every
 * |value| <= 2^27) and int32 in exact power-of-two units (scaled: every value of the lane a multiple of
 * 2^k, |value| >> k <= 2^29); wide + narrow + scaled == n_lanes */
int bs_fit_shape(bs_engine* e, uint32_t* wide, uint32_t* narrow, uint32_t* scaled);
/* per lane of the last evaluation's fit kernel: kind[d] 0 wide / 1 narrow / 2 scaled, unit[d] = k of a scaled lane
 * (0 otherwise); BS_E_STATE before the first evaluation */
int bs_fit_lanes(bs_engine* e, uint8_t* kind /*[n_lanes]*/, uint8_t* unit /*[n_lanes]*/);
/* what the last evaluation's queue sort launched: kernel 0 none (both tables empty), 1 the single-CTA kernel
 * (max(n_pods, n_groups) <= 16384), 2 the persistent kernel's lean build (4 keys in flight per thread, beside a long
 * fit kernel), 3 its wide build (16 in flight); the grid in CTAs (4096-key tiles are shared out round-robin when there
 * are more tiles than CTAs); and the radix passes kept for the group and the pod table, one per key byte that varies
 * over the table.  BS_E_STATE before the first evaluation. */
int bs_sort_shape(bs_engine* e, uint32_t* kernel, uint32_t* grid, uint32_t* group_passes, uint32_t* pod_passes);
/* the regime of the last bs_replay / bs_replay_priority walk (also one that returned BS_E_REF_PANIC): cached 1 when
 * the cluster check kept per-block summaries (fitmask, every running sum below 2^62, 1 <= n_blocks <= 1024),
 * fitmask 1 when n_rep <= 32 representative classes had a checkFit bit per node, n_blocks = ceil(n_nodes / 1024),
 * findMaxPG's n_buckets buckets of bucket_size = 32 * ceil(n_groups / 32768) groups, the walk's final lo (the leading
 * nodes the node choice stopped visiting because no pod of the table can fit there again) and monotone 1 when no pod
 * of the table has a negative cpu, memory or ephemeral-storage request (the only case lo advances).  BS_E_STATE
 * before the first walk. */
int bs_replay_shape(bs_engine* e, uint32_t* cached, uint32_t* fitmask, uint32_t* n_rep, uint32_t* n_blocks,
                    uint32_t* bucket_size, uint32_t* n_buckets, uint32_t* lo, uint32_t* monotone);

#ifdef __cplusplus
}
#endif
#endif /* BSCHED_H */
