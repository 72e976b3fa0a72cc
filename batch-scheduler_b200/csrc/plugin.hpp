// plugin.hpp — C++ host mirror of the reference's plugin surface for the hot path.
//
// The reference is Go; this image has no Go toolchain, so (per the tier rules) the host side above
// the C ABI is C++ for a compiled reference: the same names, argument meaning and status / error
// behaviour as
//   batchSchedulingPlugin.PreFilter / Permit / Less   pkg/scheduler/batch/batchscheduler.go:102,165,214
//   ScheduleOperation.AddToDenyCache                  pkg/scheduler/core/core.go:423
//   PGStatusCache.Set / Delete                        pkg/scheduler/cache/cache.go:94-120
// plus the SNAPSHOT PACKER (SURVEY.md §8(f) row 1): NodeInfo / Pod / PodGroup objects -> the SoA
// tables of include/bsched.h (resource.Quantity -> int64 lanes, labels / taints / selectors /
// tolerations -> bit sets, label -> group index, bare-name rank).
//
// Everything here is packing and bookkeeping; every decision comes from the CUDA engine through
// the C ABI (bs_evaluate, bs_prefilter, bs_permit, bs_less).
#pragma once
#include <cstdint>
#include <map>
#include <mutex>
#include <cstring>
#include <string>
#include <unordered_map>
#include <utility>
#include <vector>

#include "../../include/bsched.h"

namespace bsched {

// v1.ResourceList with quantities in their textual form ("1", "900m", "140Mi", "1e3")
using ResourceList = std::vector<std::pair<std::string, std::string>>;

constexpr const char* kPodGroupLabel = "group.batch.scheduler.tencent.com";  // pkg/util/types.go:25

// v1.ContainerPort: the fields PodFitsHostPorts reads (HostPort; ContainerPort is what hostNetwork defaults it from)
struct ContainerPort {
  std::string host_ip;      // "" = "0.0.0.0"
  std::string protocol;     // "" = "TCP"
  int32_t host_port = 0;    // <= 0: not a host port
  int32_t container_port = 0;
};
struct Container {
  bool has_limits = false;  // Resources.Limits != nil  (core.go:765)
  ResourceList limits;
  ResourceList requests;
  std::string image;        // Spec.Containers[].Image as written (ImageLocality normalizes it)
  std::vector<ContainerPort> ports;   // Spec.Containers[].Ports (init containers are not Containers)
};
struct Toleration {
  std::string key, op /* "", "Equal", "Exists" */, value, effect;
};
struct Taint {
  std::string key, value, effect;  // effect: NoSchedule | PreferNoSchedule | NoExecute
};
// v1.NodeSelectorRequirement / v1.NodeSelectorTerm: the REQUIRED node affinity of a pod
// (Spec.Affinity.NodeAffinity.RequiredDuringSchedulingIgnoredDuringExecution.NodeSelectorTerms), which
// predicates.PodMatchNodeSelector evaluates next to Spec.NodeSelector (checkFit, core.go:741-746).
struct NodeSelectorRequirement {
  std::string key, op /* In | NotIn | Exists | DoesNotExist | Gt | Lt */;
  std::vector<std::string> values;
};
struct NodeSelectorTerm {
  std::vector<NodeSelectorRequirement> match_expressions;  // against node labels
  std::vector<NodeSelectorRequirement> match_fields;       // against node fields (metadata.name)
};
// v1.PreferredSchedulingTerm: one term of Spec.Affinity.NodeAffinity.PreferredDuringSchedulingIgnoredDuringExecution,
// which kube-scheduler's NodeAffinity priority sums by weight over the nodes its preference matches
struct PreferredSchedulingTerm {
  int32_t weight = 0;               // 1..100 upstream; a term of weight 0 is skipped
  NodeSelectorTerm preference;      // only match_expressions are read; an empty list matches nothing
};
// metav1.LabelSelectorRequirement / metav1.LabelSelector: the selectors of ReplicaSets and StatefulSets
// (SelectorSpread) and of pod-affinity terms (InterPodAffinity).  An In / NotIn requirement without values, an Exists / DoesNotExist one with values, or another
// operator fails LabelSelectorAsSelector.
struct LabelSelectorRequirement {
  std::string key, op /* In | NotIn | Exists | DoesNotExist */;
  std::vector<std::string> values;
};
struct LabelSelector {
  std::map<std::string, std::string> match_labels;
  std::vector<LabelSelectorRequirement> match_expressions;
};
// v1.PodAffinityTerm (InterPodAffinity): has_selector = false is a nil selector, which matches no pod; an empty one
// matches every pod.  An empty namespaces list means the namespace of the pod that defines the term.
struct PodAffinityTerm {
  LabelSelector selector;
  bool has_selector = false;
  std::vector<std::string> namespaces;
  std::string topology_key;
};
// v1.WeightedPodAffinityTerm: one preferred pod-affinity or pod-anti-affinity term and its weight (1..100 upstream)
struct WeightedPodAffinityTerm {
  int32_t weight = 0;
  PodAffinityTerm term;
};
struct Pod {
  std::string ns, name, uid;
  std::map<std::string, std::string> labels;
  std::map<std::string, std::string> node_selector;
  bool has_required_affinity = false;                 // the required node-affinity field is non-nil
  std::vector<NodeSelectorTerm> required_affinity;    // its terms, ORed; an empty term matches nothing
  std::vector<PreferredSchedulingTerm> preferred_affinity;   // the PREFERRED node-affinity terms (NodeAffinity priority)
  std::vector<Toleration> tolerations;
  std::vector<Container> containers;
  std::vector<std::string> owner_uids;  // OwnerReferences[].UID (core.go:483-485)
  int32_t priority = 0;                 // podutil.GetPodPriority
  int64_t queue_ts_ns = 0;              // framework.PodInfo.Timestamp
  int64_t start_ns = 0;                 // Status.StartTime of a bound pod (preemption: MoreImportantPod)
  std::string controller_kind, controller_uid;   // metav1.GetControllerOf: the controlling owner ("" = none)
  bool terminating = false;             // DeletionTimestamp != nil (SelectorSpread does not count the pod)
  // Spec.Affinity.PodAffinity / PodAntiAffinity: the required pod-affinity terms (InterPodAffinity's hard weight and
  // the MatchInterPodAffinity filter), the required pod-anti-affinity terms (the filter) and the preferred
  // pod-affinity and pod-anti-affinity terms (InterPodAffinity)
  std::vector<PodAffinityTerm> required_pod_affinity, required_pod_anti_affinity;
  std::vector<WeightedPodAffinityTerm> preferred_pod_affinity, preferred_pod_anti_affinity;
};
// The objects whose selectors SelectorSpread spreads by: Services and ReplicationControllers select with a map,
// ReplicaSets and StatefulSets with a LabelSelector.  has_selector = false is a nil selector, kept distinct from an
// empty one (an empty Service selector matches every pod; an empty RC, RS or StatefulSet selector matches none).
struct Service {
  std::string ns, name;
  bool has_selector = false;
  std::map<std::string, std::string> selector;
};
struct ReplicationController {
  std::string ns, name;
  bool has_selector = false;
  std::map<std::string, std::string> selector;
};
struct ReplicaSet {
  std::string ns, name;
  bool has_selector = false;
  LabelSelector selector;
};
struct StatefulSet {
  std::string ns, name;
  bool has_selector = false;
  LabelSelector selector;
};
// what the Service, ReplicationController, ReplicaSet and StatefulSet listers hold (SetSpreadSelectors)
struct SpreadSelectors {
  std::vector<Service> services;
  std::vector<ReplicationController> controllers;
  std::vector<ReplicaSet> replica_sets;
  std::vector<StatefulSet> stateful_sets;
};
// policy/v1beta1.PodDisruptionBudget as preemption reads it (filterPodsWithPDBViolation, k8s v1.17.5 [upstream, from
// memory]): has_selector = false is a nil selector.  A nil or empty selector, or one that fails
// LabelSelectorAsSelector, matches no pod.  disruptions_allowed is Status.PodDisruptionsAllowed.
struct PodDisruptionBudget {
  std::string ns, name;
  bool has_selector = false;
  LabelSelector selector;
  int32_t disruptions_allowed = 0;
};
// v1.ContainerImage: one entry of Status.Images, the names it is known by and its size (ImageLocality)
struct ContainerImage {
  std::vector<std::string> names;
  int64_t size_bytes = 0;
};
// v1.PodSignature.PodController of one entry of the scheduler.alpha.kubernetes.io/preferAvoidPods annotation
// (NodePreferAvoidPods); the adapter parses the annotation (v1helper.GetAvoidPodsFromNodeAnnotations), an annotation
// that fails to parse giving no entries
struct PodController {
  std::string kind, uid;
};
struct Node {
  std::string name;
  std::map<std::string, std::string> labels;
  std::vector<Taint> taints;
  ResourceList allocatable;
  bool unschedulable = false;
  std::vector<ContainerImage> images;             // Status.Images
  std::vector<PodController> prefer_avoid_pods;   // the preferAvoidPods annotation's controllers
};
struct NodeInfo {          // k8s.io/kubernetes/pkg/scheduler/nodeinfo.NodeInfo, the fields core.go reads
  const Node* node = nullptr;  // nullptr: info.Node() == nil (core.go:610)
  ResourceList requested;      // info.RequestedResource()
  int32_t num_pods = 0;        // len(info.Pods())
  bool taints_error = false;   // info.Taints() returned an error (core.go:639)
  std::vector<const Pod*> pods;   // info.Pods(): the pods bound to the node, what preemption may evict (may be empty)
  std::vector<ContainerPort> used_ports;   // info.UsedPorts() flattened, as the caller supplies it (not derived from pods)
};
struct PodGroup {          // pkg/apis/podgroup/v1/types.go:62-130 (fields on the path)
  std::string ns, name;
  uint32_t min_member = 0;
  bool has_min_resources = false;
  ResourceList min_resources;
  int64_t max_schedule_time_ns = -1;  // Spec.MaxScheduleTime, <0 unset
  uint32_t scheduled = 0;             // Status.Scheduled
  std::string occupied_by;            // Status.OccupiedBy
  int64_t creation_ns = 0;
  std::string phase;                  // Status.Phase ("Scheduled" / "Running" lock its pods against preemption, core.go:235-236)
};

struct Status {  // framework.Status
  int code = BS_CODE_SUCCESS;
  std::string message;
  bool ok() const { return code == BS_CODE_SUCCESS; }
};

// resource.Quantity: exact parse of the textual form; value in units of 10^-3 (milli), rounded up
// like Quantity.MilliValue(); Value() = ceil(milli / 1000).  Returns false on a malformed string.
bool ParseQuantityMilli(const std::string& s, __int128* milli);
bool QuantityValue(const std::string& s, int64_t* out);       // Quantity.Value()
bool QuantityMilliValue(const std::string& s, int64_t* out);  // Quantity.MilliValue()
bool IsScalarResourceName(const std::string& name);           // v1helper.IsScalarResourceName
// v1helper.MatchNodeSelectorTerms (k8s v1.17.5, restated): terms are ORed, the requirements of a term ANDed;
// a term without requirements matches nothing; an invalid requirement fails its term.
bool MatchNodeSelectorTerms(const std::vector<NodeSelectorTerm>& terms, const std::map<std::string, std::string>& labels,
                            const std::string& node_name);

// The packed tables of one round (owning storage + the C-ABI views over it).
struct PackedSnapshot {
  uint32_t lanes = BS_FIXED_LANES;
  std::vector<std::string> scalar_names;  // lane 4+k
  // nodes
  std::vector<int64_t> alloc, requested;
  std::vector<int32_t> pod_count;
  std::vector<uint32_t> alloc_present, req_present;
  std::vector<uint64_t> label_mask, taint_mask;
  std::vector<uint8_t> node_flags;
  // pods
  std::vector<int64_t> req;
  std::vector<uint32_t> pod_req_present;
  std::vector<int32_t> gid, priority;
  std::vector<uint64_t> sel_mask, tol_mask;
  std::vector<int64_t> ts_ns;
  std::vector<uint8_t> pod_flags;
  // groups
  std::vector<uint32_t> min_member, scheduled, matched, min_res_present, name_rank;
  std::vector<uint8_t> group_flags;
  std::vector<int64_t> min_res, creation_ns, wait_ns;
  std::vector<uint64_t> rep_sel, rep_tol;
  uint32_t n_nodes = 0, n_pods = 0, n_groups = 0;
  // dictionaries of the round: bit b of the label / selector masks and of the taint / toleration
  // masks (needed to pack changed rows later with the same encoding, PackNodeRows)
  std::vector<std::pair<std::string, std::string>> sel_pairs;
  std::vector<Taint> taint_list;
  // affinity classes (bs_upload_affinity): pods whose node predicate does not fit the 64 selector bits —
  // required nodeAffinity terms, or every nodeSelector when the round holds more than 64 distinct pairs
  // (sel_in_table: the masks stay zero then) — share one class per distinct predicate; aff_bits holds the
  // host-evaluated verdict of every class on every node
  struct AffClassDef {
    std::map<std::string, std::string> node_selector;   // only when sel_in_table
    bool has_required_affinity = false;
    std::vector<NodeSelectorTerm> terms;
  };
  bool sel_in_table = false;
  std::vector<AffClassDef> aff_classes;
  std::vector<std::string> aff_signatures;              // canonical text of each class (lookup key)
  std::vector<uint32_t> aff_class, rep_aff;             // per pod / per group, BS_AFF_NONE = none
  std::vector<uint32_t> aff_bits;                       // [n_aff][ceil(n_nodes / 32)]
  uint32_t n_aff() const { return (uint32_t)aff_classes.size(); }

  bs_node_table node_table() const;
  bs_pod_table pod_table() const;
  bs_group_table group_table() const;
};

// The columns of the TaintToleration and preferred NodeAffinity priorities of one round (bs_upload_node_preferences,
// bs_upload_pod_preferences): the round's dictionary of distinct PreferNoSchedule taints (key, value), each node's bits
// of it and each pending pod's tolerated bits; the pods' distinct preferred-affinity classes (by the canonical text of
// their weighted terms) and the class x node table of summed weights.
struct PackedPreferences {
  std::vector<Taint> taints;                    // bit b of the masks
  std::vector<uint64_t> prefer_taints;          // [n_nodes]
  std::vector<uint64_t> prefer_tol;             // [n_pods]
  std::vector<uint32_t> pref_class;             // [n_pods], BS_PREF_NONE = no preferred term of non-zero weight
  std::vector<std::string> class_signatures;    // canonical text of each class
  std::vector<int32_t> pref_weights;            // [n_classes][n_nodes]
  uint32_t n_classes() const { return (uint32_t)class_signatures.size(); }
};

// The columns of the ImageLocality and NodePreferAvoidPods priorities of one round (bs_upload_node_locality,
// bs_upload_pod_locality): the dictionary of reported image names that some pending pod's normalized container image
// matches, with each name's size and bit row over the nodes; each pod's class (its sorted id list, deduplicated); the
// dictionary of RC / RS controllers listed on some node and controlling some pending pod, each node's bits of it and
// each pod's bit.
struct PackedLocality {
  std::vector<std::string> names;               // id i of the image dictionary
  std::vector<int64_t> image_size;              // [n_images]
  std::vector<uint32_t> image_bits;             // [n_images][ceil(n_nodes / 32)]
  std::vector<uint32_t> image_class;            // [n_pods], BS_IMAGE_NONE = no dictionary image
  std::vector<uint32_t> class_offset{0};        // [n_classes + 1]
  std::vector<uint32_t> class_images;           // [class_offset.back()]
  std::vector<PodController> controllers;       // bit b of the avoid masks
  std::vector<uint64_t> avoid_mask;             // [n_nodes]
  std::vector<uint8_t> avoid_bit;               // [n_pods], BS_AVOID_NONE = no listed RC / RS controller
  uint32_t n_classes() const { return (uint32_t)class_offset.size() - 1; }
};
// The columns of the SelectorSpread priority of one round (bs_upload_node_spread, bs_upload_pod_spread): the zone
// dictionary (GetZoneKey of each node, in order of first appearance, at most 64) and each node's zone; each pending
// pod's class (its namespace and the sorted set of its selectors' canonical texts; BS_SPREAD_NONE without selectors)
// and the class x node table of matching pods over NodeInfo::pods.
struct PackedSpread {
  std::vector<std::string> zones;               // id z of the zone dictionary
  std::vector<uint8_t> zone;                    // [n_nodes], BS_ZONE_NONE = no zone key
  std::vector<uint32_t> spread_class;           // [n_pods], BS_SPREAD_NONE = no selector
  std::vector<std::string> class_signatures;    // namespace and selector texts of each class
  std::vector<int32_t> counts;                  // [n_classes][n_nodes]
  uint32_t n_classes() const { return (uint32_t)class_signatures.size(); }
};
// The columns of the InterPodAffinity priority of one round (bs_upload_node_interpod, bs_upload_pod_interpod): the
// topology keys and each key's values in order of first appearance; the term dictionary (term_signatures: the
// resolved, sorted namespaces, the selector's canonical text and the key); the bound pods of NodeInfo::pods and their
// classes; each pending pod's class.  A class is a sorted list of (term, own, match).
struct PackedInterPodAffinity {
  struct Classes {
    std::vector<uint32_t> offset{0};            // [n_classes + 1]
    std::vector<uint32_t> term;
    std::vector<int32_t> own;
    std::vector<uint8_t> match;
    uint32_t n_classes() const { return (uint32_t)offset.size() - 1; }
  };
  std::vector<std::string> keys;                // key id -> topology key
  std::vector<std::vector<std::string>> values; // [key] value id -> label value
  std::vector<uint32_t> n_values;               // [n_keys]
  std::vector<uint32_t> topo;                   // [n_keys][n_nodes], BS_TOPO_NONE = the node lacks the key
  std::vector<std::string> term_signatures;     // term id -> signature
  std::vector<uint32_t> term_key;               // [n_terms]
  std::vector<uint32_t> bound_node, bound_class;   // [n_bound], BS_IPA_NONE = no entries
  Classes bound_classes;
  std::vector<uint32_t> pod_class;              // [n_pods], BS_IPA_NONE = no entries (scores 0)
  Classes pod_classes;
};
// The columns of the MatchInterPodAffinity filter of one round (bs_upload_node_interpod_filter,
// bs_upload_pod_interpod_filter): keys, values and topo as PackedInterPodAffinity numbers them; the filter's own term
// dictionary (term_signatures); the bound pods of NodeInfo::pods and their classes of (term, own, match); each pending
// pod's class of (term, role) with its self_match byte.
// The columns of the PodFitsHostPorts filter of one round (bs_upload_node_host_ports, bs_upload_pod_host_ports): the
// dictionary (ip id, protocol id, port; ip id 0 = "0.0.0.0", the other ips and the protocols numbered by first
// appearance), each node's used mask and each pending pod's want mask; with bound, each bound pod's mask too.
struct PackedHostPorts {
  std::vector<uint32_t> ip, protocol;
  std::vector<int32_t> port;
  std::vector<uint64_t> used;   // [n_nodes]
  std::vector<uint64_t> want;   // [n_pods]
  std::vector<uint64_t> bound;  // [bound pods] NodeInfo::pods in PackBoundPods' row order (bs_upload_bound_host_ports)
  std::vector<std::string> ips{"0.0.0.0"}, protocols;   // id -> text
};
struct PackedInterPodFilter {
  std::vector<std::string> keys;
  std::vector<std::vector<std::string>> values;
  std::vector<uint32_t> n_values;
  std::vector<uint32_t> topo;                   // [n_keys][n_nodes], BS_TOPO_NONE = the node lacks the key
  std::vector<std::string> term_signatures;     // term id -> signature
  std::vector<uint32_t> term_key;               // [n_terms]
  std::vector<uint32_t> bound_node, bound_class;   // [n_bound], BS_IPF_NONE = no entries
  PackedInterPodAffinity::Classes bound_classes;
  std::vector<uint32_t> pod_class;              // [n_pods], BS_IPF_NONE = no entries (passes every node)
  std::vector<uint32_t> pod_offset{0};          // [n_classes + 1]
  std::vector<uint32_t> pod_term;
  std::vector<uint8_t> pod_role;                // BS_IPF_AFFINITY / BS_IPF_ANTI / BS_IPF_EXISTING
  std::vector<uint8_t> self_match;              // [n_classes]
  uint32_t n_pod_classes() const { return (uint32_t)pod_offset.size() - 1; }
  // the placed side (bs_upload_pod_interpod_placed), packed only on request: what each pending pod adds to presence
  // once a walk assumes it, as a bound pod's class
  std::vector<uint32_t> placed_class;           // [n_pods], BS_IPF_NONE = no entries; empty when not packed
  PackedInterPodAffinity::Classes placed_classes;
};
// normalizedImageName (ImageLocality): ":latest" appended when the last ':' does not follow the last '/'
std::string normalized_image_name(const std::string& name);

// string -> row index of one round, built in one go: the keys are copied into ONE arena (no allocation per key),
// hashed in parallel, and a later duplicate overwrites an earlier one, as `map[key] = row` in a loop would.
// Lookups are exact (the arena bytes are compared), not by hash alone.
// The bound-pod table of a round (bs_bound_table): every pod NodeInfo.Pods() lists, in snapshot order.
struct PackedBound {
  uint32_t lanes = BS_FIXED_LANES, n = 0;
  std::vector<uint32_t> node, req_present;
  std::vector<int64_t> req, start_ns;   // req: [lanes][n], the containers' Requests
  std::vector<int32_t> gid, priority;
  std::vector<uint8_t> flags;
  std::vector<const Pod*> pods;
  bs_bound_table table() const;
};

class StrIndex {
 public:
  // key_at(i) -> const std::string* (nullptr: row i has no key)
  template <class KeyAt>
  void build(size_t n, KeyAt key_at, int threads) {
    off_.assign(n + 1, 0);
    for (size_t i = 0; i < n; ++i) {
      const std::string* k = key_at(i);
      off_[i + 1] = off_[i] + (k ? k->size() + 1 : 0);   // +1: a present key owns at least one byte (empty != absent)
    }
    chars_.resize(off_[n]);
    std::vector<uint64_t> h(n);
#pragma omp parallel for num_threads(threads) schedule(static)
    for (size_t i = 0; i < n; ++i) {
      const std::string* k = key_at(i);
      if (!k) continue;
      char* dst = chars_.data() + off_[i];
      std::memcpy(dst, k->data(), k->size());
      dst[k->size()] = 0;
      h[i] = hash(k->data(), k->size());
    }
    size_t cap = 16;
    while (cap < 2 * n) cap <<= 1;
    slot_.assign(cap, kNone);
    mask_ = (uint32_t)(cap - 1);
    for (size_t i = 0; i < n; ++i) {
      if (off_[i + 1] == off_[i]) continue;
      uint32_t s = (uint32_t)h[i] & mask_;
      while (slot_[s] != kNone && !equal(slot_[s], chars_.data() + off_[i], off_[i + 1] - off_[i] - 1)) s = (s + 1) & mask_;
      slot_[s] = (uint32_t)i;   // empty slot, or the same key again: the later row wins
    }
  }
  int32_t find(const std::string& k) const {
    if (slot_.empty()) return -1;
    uint32_t s = (uint32_t)hash(k.data(), k.size()) & mask_;
    while (slot_[s] != kNone) {
      if (equal(slot_[s], k.data(), k.size())) return (int32_t)slot_[s];
      s = (s + 1) & mask_;
    }
    return -1;
  }
  void clear() { off_.clear(); chars_.clear(); slot_.clear(); mask_ = 0; }

 private:
  static constexpr uint32_t kNone = 0xffffffffu;
  static uint64_t hash(const char* p, size_t n) {
    uint64_t h = 1469598103934665603ull;
    for (size_t i = 0; i < n; ++i) { h ^= (unsigned char)p[i]; h *= 1099511628211ull; }
    return h ^ (h >> 32);
  }
  bool equal(uint32_t row, const char* p, size_t n) const {
    return off_[row + 1] - off_[row] - 1 == n && std::memcmp(chars_.data() + off_[row], p, n) == 0;
  }
  std::vector<size_t> off_;
  std::vector<char> chars_;
  std::vector<uint32_t> slot_;
  uint32_t mask_ = 0;
};

class BatchSchedulingPlugin {
 public:
  // batch.New (batchscheduler.go:377): max_schedule_time from the plugin args (Configuration, :71-75)
  // topk > 0 adds BS_OUT_TOPK: each round also keeps every pending pod's topk best fitting nodes (TopNodes)
  // priority_k > 0 adds BS_OUT_PRIORITY: each round also keeps every pending pod's priority_k best fitting nodes under
  // kube-scheduler's resource priorities (PriorityNodes); with topk too, the two must be equal (else init_error())
  BatchSchedulingPlugin(int device, int64_t max_schedule_time_ns, uint32_t out_flags = BS_OUT_FIT_BITMAP, uint32_t topk = 0,
                        uint32_t priority_k = 0);
  ~BatchSchedulingPlugin();
  BatchSchedulingPlugin(const BatchSchedulingPlugin&) = delete;
  BatchSchedulingPlugin& operator=(const BatchSchedulingPlugin&) = delete;
  const std::string& init_error() const { return init_error_; }

  // PGStatusCache.Set / Delete (cache.go:104-120), keyed by "namespace/name"
  void SetPodGroup(const PodGroup& pg);
  void DeletePodGroup(const std::string& ns_name);

  // One scheduling round: pack the snapshot (list order preserved, core.go:597,604) and the pending
  // pods (queue arrival order), upload, evaluate on the GPU, fetch.  now_ns drives TTL expiry.
  Status BeginRound(const std::vector<const NodeInfo*>& snapshot, const std::vector<const Pod*>& pending,
                    int64_t now_ns);

  // batchSchedulingPlugin.PreFilter (batchscheduler.go:102-108)
  Status PreFilter(const Pod& pod);
  // batchSchedulingPlugin.Permit (batchscheduler.go:165-202): status + wait duration (ns)
  std::pair<Status, int64_t> Permit(const Pod& pod, const std::string& node_name, bool* start_signal = nullptr);
  // batchSchedulingPlugin.Less (batchscheduler.go:214-216)
  bool Less(const Pod& a, const Pod& b);
  // batchSchedulingPlugin.Filter (batchscheduler.go:151-157) -> core.Filter (core.go:170-191); the
  // plugin must have been created with BS_OUT_FILTER in out_flags.  On failure the group is
  // deny-listed (core.go:184), on success the pod is remembered as permitted for 2 s (:188).
  Status Filter(const Pod& pod, const std::string& node_name);
  // ScheduleOperation.AddToDenyCache (core.go:423-425): 20 s, Add semantics (no-op if present)
  void AddToDenyCache(const std::string& ns_name, int64_t now_ns);
  // lastPermittedPod.Add(uid, 2s) (core.go:188)
  void AddPermitted(const std::string& uid, int64_t now_ns);
  // One janitor tick of the gangs' TTL tables (controller.go:322-333 via bs_expire): a gang whose wait time ran
  // out rejects every pod it still holds at Permit ("Group failed", batchscheduler.go:347-354) and is deny-listed
  // for 20 s.  rejected: uids to Reject; evicted: the groups ("namespace/name").
  Status Tick(int64_t now_ns, std::vector<std::string>* rejected_uids, std::vector<std::string>* evicted_groups);
  // StartBatchSchedule's Allow loop (batchscheduler.go:292-344) for a group whose Permit fired the start signal:
  // (uid, node name) of every waiting pod to Allow; empty while the gang is incomplete.
  Status AllowList(const std::string& ns_name, int64_t now_ns, std::vector<std::pair<std::string, std::string>>* allow);
  static uint64_t IdOf(const std::string& s);   // FNV-1a 64: uids and "ns/name"s cross the C ABI as ids

  // The whole pending queue of the last BeginRound walked through the reference's pod-at-a-time cycle
  // (PreFilter against live state -> node choice -> assume -> Permit, core.go:88-167,268-309)
  // on the device, in the order Less defines (bs_replay; SURVEY 8(f) row 4).  A what-if: neither the
  // plugin's caches nor the uploaded tables change.  out is indexed like `pending`.
  struct ReplayDecision {
    uint8_t prefilter = 0;    // bs_prefilter_code
    int32_t node = -1;        // snapshot index of the node the pod was assumed onto, -1 none
    bool ready = false;       // Permit found the gang complete with this pod (core.go:303)
    uint32_t position = 0;    // place in the walked queue
  };
  // where the walk places a pod that passes PreFilter
  enum class ReplayNodeChoice {
    kFirstFit,   // the first fitting node in snapshot order (bs_replay)
    kPriority,   // the best fitting node under the resource priorities (SetScoreWeights) on the live state
                 // (bs_replay_priority); needs a plugin created with priority_k > 0, whose rounds upload the non-zero
                 // request columns; otherwise ReplayQueue returns an error
  };
  Status ReplayQueue(std::vector<ReplayDecision>* out, ReplayNodeChoice choice = ReplayNodeChoice::kFirstFit);

  // results of the last round, by pending index
  const PackedSnapshot& packed() const { return packed_; }
  const std::vector<uint8_t>& prefilter_codes() const { return prefilter_; }
  const std::vector<uint8_t>& admit_codes() const { return admit_; }
  const std::vector<uint32_t>& queue_order() const { return order_; }
  const std::vector<uint32_t>& feasible_counts() const { return feasible_; }
  const std::vector<int32_t>& best_nodes() const { return best_node_; }
  // the pod's best fitting nodes of the last round (plugin created with topk > 0): (node name, residual score),
  // score descending, then snapshot order; at most topk of them, empty for an unknown uid
  std::vector<std::pair<std::string, int64_t>> TopNodes(const std::string& uid) const;
  // plugin created with BS_OUT_REASONS in out_flags: the pod's reason row of the last round, 4 + lanes counters in the
  // bins of BS_REASON_* (empty for an unknown uid), and the FailedScheduling message built from it
  // ("0/N nodes are available: ..."; lanes >= 4 by their resource names) for a pod that fits no node, "" otherwise
  std::vector<uint32_t> ReasonCounts(const std::string& uid) const;
  std::string FitError(const std::string& uid) const;
  // plugin created with priority_k > 0: the pod's best fitting nodes of the last round under the resource priorities
  // (node name, score), score descending, then snapshot order; at most priority_k of them, empty for an unknown uid.
  // Entry 0 is where kube-scheduler's default profile would bind the pod, as far as these priorities decide it.
  std::vector<std::pair<std::string, int64_t>> PriorityNodes(const std::string& uid) const;
  // weights of NodeResourcesLeastAllocated, NodeResourcesMostAllocated and NodeResourcesBalancedAllocation (default
  // 1, 0, 1), from the next round or delta round on
  void SetScoreWeights(uint32_t least, uint32_t most, uint32_t balanced);
  // kube-scheduler v1.17's RequestedToCapacityRatio priority (bs_set_ratio_priority), added to PriorityNodes and
  // ReplayQueue(kPriority) with `weight` (0 = off, the default), from the next round or delta round on.  `shape` holds
  // (utilization 0..100, score 0..10) points as the policy file gives them, utilization strictly ascending; the scores
  // are multiplied by 10 (MaxNodeScore / MaxCustomPriorityScore).  `resources` maps a resource name to a weight in
  // 1..100; empty means cpu 1, memory 1.  Every round maps the names onto its lanes: cpu, memory and ephemeral-storage
  // to lanes 0-2, a scalar resource of the round to its lane, and `pods` or a name no node of the round carries to the
  // weight of resources with capacity 0 everywhere.  An invalid setting returns an error and the previous one stays.
  Status SetRatioPriority(uint32_t weight, const std::vector<std::pair<uint32_t, uint32_t>>& shape,
                          const std::map<std::string, uint32_t>& resources);
  // weights of kube-scheduler v1.17's TaintToleration and preferred NodeAffinity priorities in PriorityNodes
  // (bs_set_node_priority_weights; 0, 0 = off, the default; v1.17's default profile is 1, 1), from the next round or
  // delta round on, on a plugin created with priority_k > 0.  While either is non-zero, ReplayQueue(kPriority) returns
  // an error.
  void SetNodePriorityWeights(uint32_t taint_toleration, uint32_t node_affinity);
  // weights of kube-scheduler v1.17's ImageLocality and NodePreferAvoidPods priorities in PriorityNodes and in
  // ReplayQueue(kPriority) (bs_set_locality_weights; 0, 0 = off, the default; v1.17's default profile is 1, 10000),
  // from the next round or delta round on, on a plugin created with priority_k > 0.
  void SetLocalityWeights(uint32_t image_locality, uint32_t prefer_avoid_pods);
  // the content of the Service, ReplicationController, ReplicaSet and StatefulSet listers, read by the next round
  void SetSpreadSelectors(SpreadSelectors selectors);
  // the content of the PodDisruptionBudget lister, read when the bound-pod table is packed next: at the next
  // BeginRound, UpdateNodes or UpdateGroups (PackBoundPods sets BS_BOUND_PDB_VIOLATING from it)
  void SetPodDisruptionBudgets(std::vector<PodDisruptionBudget> pdbs);
  // weight of kube-scheduler v1.17's SelectorSpread priority in PriorityNodes (bs_set_spread_weight; 0 = off, the
  // default; v1.17's default profile is 1), read by the next round; ReplayQueue(kPriority) refuses a non-zero weight
  void SetSelectorSpreadWeight(uint32_t selector_spread);
  // weight of kube-scheduler v1.17's InterPodAffinity priority in PriorityNodes (bs_set_interpod_weight; 0 = off, the
  // default; v1.17's default profile is 1), read by the next round; ReplayQueue(kPriority) refuses a non-zero weight
  void SetInterPodAffinityWeight(uint32_t inter_pod_affinity);
  // kube-scheduler v1.17's MatchInterPodAffinity filter in every pod's fit set (bs_set_interpod_filter; off by
  // default), from the next round, delta round or UpdateNodes on: PackInterPodFilter's columns are uploaded with each
  // of them.  While it is on, Preempt, PreemptAll and PreemptQueue return an error, and so does ReplayQueue unless
  // SetInterPodAffinityFilterInWalks is on.
  void SetInterPodAffinityFilter(bool on);
  // the MatchInterPodAffinity filter in ReplayQueue as well (off by default): while this and the filter are on, the
  // next round, delta round or UpdateNodes packs and uploads the pending pods' placed classes too
  // (PackInterPodFilter(..., placed = true), bs_upload_pod_interpod_placed), and ReplayQueue (both choices) walks under
  // the filter on presence that follows its own placements.  Off, the rounds pack and upload what they did before.
  void SetInterPodAffinityFilterInWalks(bool on);
  // kube-scheduler v1.17's PodFitsHostPorts filter in every pod's fit set and in ReplayQueue (bs_set_host_port_filter;
  // off by default), from the next round, delta round or UpdateNodes on: PackHostPorts' columns are uploaded with each
  // of them.  While it is on, Preempt, PreemptAll and PreemptQueue return an error unless
  // SetHostPortFilterInPreemption is on too.
  void SetHostPortFilter(bool on);
  // the PodFitsHostPorts filter in preemption as well (off by default): while this and the filter are on, every upload
  // of the bound-pod table and of the filter's sides is followed by the bound pods' host-port masks
  // (PackHostPorts(..., bound = true), bs_upload_bound_host_ports), from the next round, delta round or UpdateNodes
  // on, and Preempt, PreemptAll and PreemptQueue run under the filter.  Off, the rounds pack and upload what they did
  // before and the three calls refuse under the filter.
  void SetHostPortFilterInPreemption(bool on);
  // the last round's host-port companion count of a pending pod (bs_fetch_host_port_reason_rows); empty without
  // BS_OUT_REASONS, while the filter is off or for an unknown uid
  std::vector<uint32_t> HostPortReasonCounts(const std::string& uid) const;
  // the last round's companion reason row of a pending pod (bs_fetch_interpod_reason_rows: the nodes that pass every
  // other check and fail the filter at E, A, N); empty without BS_OUT_REASONS or for an unknown uid
  std::vector<uint32_t> InterPodReasonCounts(const std::string& uid) const;
  // hardPodAffinitySymmetricWeight: the weight of a bound pod's required pod-affinity term in InterPodAffinity,
  // 0..100 (else an error), default 1; 0 leaves those terms out
  Status SetHardPodAffinityWeight(int32_t hard_pod_affinity_weight);
  int group_index(const std::string& ns_name) const;
  double last_pack_ms() const { return last_pack_ms_; }
  double last_device_ms() const { return last_device_ms_; }
  bs_engine* engine() const { return eng_; }

  // Incremental snapshot update (SURVEY 8(f) row 1): between cycles the informer touches a few
  // NodeInfos.  PackNodeRows re-packs just those with the encoding of the last full pack (`ctx`) into
  // a compact node table; *needs_full is set when a row brings a scalar resource or a NoSchedule /
  // NoExecute taint the dictionaries of `ctx` do not hold (then only a full Pack is correct).
  // UpdateNodes does that for the current round and scatters the rows into the resident device
  // table (bs_update_nodes); `changed` pairs the snapshot index with the new NodeInfo.
  static Status PackNodeRows(const PackedSnapshot& ctx, const std::vector<const NodeInfo*>& rows, PackedSnapshot* out,
                             bool* needs_full);
  Status UpdateNodes(const std::vector<std::pair<uint32_t, const NodeInfo*>>& changed, bool evaluate = true);
  // one delta round: the informer's changed NodeInfos and PodGroups scattered into the resident tables, then
  // ONE re-evaluation (UpdateNodes / UpdateGroups with evaluate = false, then the round)
  Status UpdateRound(const std::vector<std::pair<uint32_t, const NodeInfo*>>& changed_nodes,
                     const std::vector<std::string>& changed_groups, int64_t now_ns);
  // The same for PodGroup state (cache.go:52-67): one changed group = its table index, the object, the
  // unexpired matched count, the SCHEDULED / HAS_POD / DENIED flags and the representative pod (or null).
  // Names are immutable, so the bare-name rank is taken over from `ctx`.  needs_full: MinResources or the
  // representative pod use a scalar resource / nodeSelector pair the round's dictionaries do not hold.
  struct GroupDelta {
    uint32_t index = 0;
    const PodGroup* pg = nullptr;
    uint32_t matched = 0;
    uint8_t flags = 0;
    const Pod* rep_pod = nullptr;
  };
  static Status PackGroupRows(const PackedSnapshot& ctx, const std::vector<GroupDelta>& rows, int64_t default_wait_ns,
                              PackedSnapshot* out, bool* needs_full);
  // re-derives the named groups ("namespace/name") from the plugin's caches and scatters their rows
  // into the resident device table (bs_update_groups), then re-evaluates the round
  Status UpdateGroups(const std::vector<std::string>& ns_names, int64_t now_ns, bool evaluate = true);

  // the packer alone (no GPU): objects -> tables
  // The bound pods of `snapshot` against the lanes of `ctx`: demand = the containers' Requests (NodeInfo.RemovePod
  // subtracts what AddPod added: Requests, not Limits); gid from the group label and "ns/<label>" in group_row
  // (BS_GID_NONE without the label, BS_GID_MISSING when the group is not in the table); BS_BOUND_GROUP_LOCKED when
  // that group's row is in `locked` (Status.Phase Scheduled or Running).  BS_BOUND_PDB_VIOLATING by
  // filterPodsWithPDBViolation: the pod has a label and some budget of `pdbs` in its namespace, with a selector that
  // converts, is not empty and matches the pod's labels, allows <= 0 disruptions.
  static Status PackBoundPods(const PackedSnapshot& ctx, const std::vector<const NodeInfo*>& snapshot,
                              const std::unordered_map<std::string, uint32_t>& group_row,
                              const std::vector<uint8_t>& locked, PackedBound* out,
                              const std::vector<PodDisruptionBudget>& pdbs = {});
  // batchSchedulingPluginExtension.RemovePod (batchscheduler.go:132-144) -> core.PreemptRemovePod (core.go:203-260):
  // the preemptor must be a pending pod of the round, the victim a pod some NodeInfo of the round lists
  Status RemovePod(const Pod& preemptor, const Pod& victim);
  // PreemptAddPod always succeeds (core.go:194-196)
  Status AddPod(const Pod&, const Pod&) { return Status{}; }
  // genericScheduler.Preempt for one pending pod of the round against the round's snapshot: the node preemption would
  // pick ("" none) and the uids of the pods it would evict there: those that violate a PodDisruptionBudget
  // (SetPodDisruptionBudgets) first, then the others, each part most important first
  Status Preempt(const std::string& uid, std::string* node, std::vector<std::string>* victim_uids);
  struct Preemption {
    std::string uid, node;
    std::vector<std::string> victims;
  };
  // Preempt for every pending pod that passed PreFilter and fits no node (upstream preempts only on a FitError), the
  // victims in Preempt's order
  Status PreemptAll(std::vector<Preemption>* out);
  // PreemptAll's pods as kube-scheduler preempts them, one per cycle (bs_preempt_walk): in the round's queue_order(),
  // each seeing the evictions and nominations of those before it.  With `gang`, each group's later preemptors move up
  // to its first one (the order is kept otherwise) and a group gets nodes for all its preemptors or for none; a group
  // whose preemptors have different priorities is an error.  Entries in walk order; a rolled-back member has node "".
  Status PreemptQueue(std::vector<Preemption>* out, bool gang);
  const PackedBound& bound() const { return bound_; }
  // The non-zero request columns of the resource priorities (no GPU): per pending pod and per NodeInfo (over
  // NodeInfo::pods), [2][n] int64 — cpu millicores, memory bytes — summed over the containers' Requests, a container
  // without a cpu key counting 100 m and without a memory key 200 MiB (an explicit zero stays zero).  Init containers
  // and pod overhead are not modelled.
  static Status PackNonZero(const std::vector<const NodeInfo*>& snapshot, const std::vector<const Pod*>& pending,
                            std::vector<int64_t>* node_nz, std::vector<int64_t>* pod_nz);
  // The columns of the TaintToleration and preferred NodeAffinity priorities (no GPU): a node's PreferNoSchedule taints
  // as bits of the round's dictionary (more than 64 distinct ones is an error); a pod tolerates a bit when one of its
  // tolerations with an empty or PreferNoSchedule effect tolerates the taint (ToleratesTaint); a class's weight on a
  // node sums the weights of its terms whose match_expressions all match the node's labels.  A term with an invalid
  // requirement counts 0 there (upstream, it fails the pod's scoring); a negative weight is an error.
  static Status PackPreferences(const std::vector<const NodeInfo*>& snapshot, const std::vector<const Pod*>& pending,
                                PackedPreferences* out);
  // The columns of the ImageLocality and NodePreferAvoidPods priorities (no GPU).  Only Spec.Containers count; a name
  // reported with different sizes takes the size of the lowest node index reporting it; a controller of a kind other
  // than ReplicationController / ReplicaSet counts as none.  More than BS_LOC_CLASS_MAX dictionary images in one pod,
  // or more than 64 controllers in the avoid dictionary, is an error.
  static Status PackLocality(const std::vector<const NodeInfo*>& snapshot, const std::vector<const Pod*>& pending,
                             PackedLocality* out);
  // The columns of the SelectorSpread priority (no GPU).  A pod's selectors are those of getSelectors: the Services of
  // its namespace whose non-nil selector matches its labels, and, when it has labels, the RCs, ReplicaSets and
  // StatefulSets of its namespace whose non-empty selector matches them (a selector that fails to convert is
  // skipped).  count(class, node) = the pods of NodeInfo::pods in the class's namespace, not terminating, that every
  // selector matches.  More than 64 zones, or a count above BS_SPREAD_COUNT_MAX, is an error.
  static Status PackSpread(const std::vector<const NodeInfo*>& snapshot, const std::vector<const Pod*>& pending,
                           const SpreadSelectors& selectors, PackedSpread* out);
  // The columns of the InterPodAffinity priority (no GPU), from NodeInfo::pods (terminating ones too) and the pending
  // pods.  Keys and terms are numbered in order of first appearance over the bound pods' terms (required affinity
  // while hard_weight > 0, preferred affinity, preferred anti-affinity), then the pending pods' (preferred affinity,
  // preferred anti-affinity); a term is identified by its resolved, sorted namespaces, its converted selector's
  // canonical text (SelectorSpread's conversion) and its key.  A term with an empty key matches no node and is left
  // out; so is a term whose selector fails to convert.  Each key's values are numbered in order of first appearance
  // over the nodes.  A pod lists (t, own, match) for every term it owns (own: its summed signed weights, +hard_weight
  // per required term of a bound pod) or matches among the other side's terms; a pod without entries has no class,
  // and classes are numbered in order of first appearance.  A pending pod gets no class (BS_IPA_NONE, score 0), as
  // upstream fails its score, when a processed term of a bound pod fails to convert, or when one of its own terms does
  // and a pod is bound.  More than BS_IPA_KEY_MAX keys, BS_IPA_BOUND_MAX bound pods or BS_IPA_CLASS_MAX entries in a
  // class, or an own outside BS_IPA_OWN_MAX, is an error.
  static Status PackInterPodAffinity(const std::vector<const NodeInfo*>& snapshot,
                                     const std::vector<const Pod*>& pending, int32_t hard_weight,
                                     PackedInterPodAffinity* out);

  // The columns of the MatchInterPodAffinity filter (no GPU), from NodeInfo::pods of nodes with a Node() (terminating
  // ones too) and the pending pods.  Keys and values are numbered as PackInterPodAffinity numbers them, and terms are
  // identified the same way (resolved, sorted namespaces, SelectorSpread's converted selector text, key).  The
  // dictionary: the bound pods' required anti-affinity terms (own = 1 on their owners; a pending pod that matches one
  // lists it as BS_IPF_EXISTING), then per pending pod its required affinity set, one term per set member
  // (BS_IPF_AFFINITY; a bound pod's match = it matches every member), and its required anti-affinity terms
  // (BS_IPF_ANTI; match = it matches the term); equal sets and equal anti terms share their terms.  A selector that
  // fails to convert matches no pod; an empty key is a key no node carries.  self_match: the pending pod matches its
  // whole set.  Classes are numbered in order of first appearance; a pod without entries has none (BS_IPF_NONE).
  // With `placed`, also each pending pod's placed class over the same dictionary: own = 1 on its required
  // anti-affinity terms, match = 1 on the bound pods' anti-affinity terms it matches, on every term of each affinity set
  // it matches as a whole (its own included) and on each pending anti-affinity term it matches (P x terms selector
  // matching, hence on request).  Its match entries on bound pods' terms are exactly its BS_IPF_EXISTING entries.
  // More than BS_IPA_KEY_MAX keys, BS_IPF_BOUND_MAX bound pods or BS_IPF_CLASS_MAX entries in a class is an error.
  static Status PackInterPodFilter(const std::vector<const NodeInfo*>& snapshot, const std::vector<const Pod*>& pending,
                                   PackedInterPodFilter* out, bool placed = false);
  // PodFitsHostPorts' columns: HostPortInfo's sanitizing (port <= 0 dropped, "" ip = "0.0.0.0", "" protocol = "TCP");
  // the dictionary holds the pending pods' wanted (ip, protocol, port) in order of first appearance, then the nodes'
  // used ones that conflict with one of them (a used entry that conflicts with nothing wanted never decides a verdict).
  // More than BS_HOSTPORT_MAX entries is an error.  bound: also each NodeInfo::pods row's mask from its
  // Container::ports, sanitized the same way, with the bit of the dictionary entry each port equals (a port in no
  // entry conflicts with no pending pod and is left out).
  static Status PackHostPorts(const std::vector<const NodeInfo*>& snapshot, const std::vector<const Pod*>& pending,
                              PackedHostPorts* out, bool bound = false);

  static Status Pack(const std::vector<const NodeInfo*>& snapshot, const std::vector<const Pod*>& pending,
                     const std::vector<PodGroup>& groups, const std::vector<uint32_t>& matched,
                     const std::vector<uint8_t>& extra_group_flags, const std::vector<uint8_t>& extra_pod_flags,
                     int64_t default_wait_ns, PackedSnapshot* out);
  // the same with each group given as a GroupDelta (object, matched count, flags, representative pod); a group's
  // row is its position in `groups`, GroupDelta::index is not read
  static Status Pack(const std::vector<const NodeInfo*>& snapshot, const std::vector<const Pod*>& pending,
                     const std::vector<GroupDelta>& groups, const std::vector<uint8_t>& extra_pod_flags,
                     int64_t default_wait_ns, PackedSnapshot* out);

 private:
  // MatchedPodNodes / PodNameUIDs / pgs.Scheduled and the deny / permitted caches live in the ENGINE (bs_state_*,
  // bs_permit_at, bs_expire, bs_allow_list: include/bsched.h "gang state"); here only what packing needs
  struct GroupState {
    PodGroup pg;
    bool has_pod = false;                                           // pgs.Pod != nil
    uint64_t rep_sel_pairs_hash = 0;
    Pod rep_pod;                                                    // pgs.Pod
  };
  bs_engine* eng_ = nullptr;
  bool state_ready_ = false;   // bs_state_reset has run for this plugin's engine lineage
  int device_ = 0;
  uint32_t out_flags_ = 0, eng_lanes_ = 0, topk_ = 0, priority_k_ = 0;
  uint32_t weights_[3] = {1, 0, 1};
  uint32_t ratio_weight_ = 0;                          // SetRatioPriority: shape in engine units, weights by name
  std::vector<uint32_t> ratio_util_{0, 100}, ratio_score_{100, 0};
  std::map<std::string, uint32_t> ratio_resources_{{"cpu", 1}, {"memory", 1}};
  uint32_t node_prio_weights_[2] = {0, 0};             // SetNodePriorityWeights: TaintToleration, NodeAffinity
  uint32_t locality_weights_[2] = {0, 0};              // SetLocalityWeights: ImageLocality, NodePreferAvoidPods
  uint32_t spread_weight_ = 0;                          // SetSelectorSpreadWeight
  SpreadSelectors spread_selectors_;                    // SetSpreadSelectors
  std::vector<PodDisruptionBudget> pdbs_;               // SetPodDisruptionBudgets
  uint32_t interpod_weight_ = 0;                        // SetInterPodAffinityWeight
  int32_t hard_pod_affinity_weight_ = 1;                // SetHardPodAffinityWeight
  bool interpod_filter_ = false;                        // SetInterPodAffinityFilter
  bool interpod_filter_walks_ = false;                  // SetInterPodAffinityFilterInWalks
  bool host_port_filter_ = false;                       // SetHostPortFilter
  bool host_port_preempt_ = false;                      // SetHostPortFilterInPreemption
  std::string init_error_;
  int64_t max_schedule_time_ns_;
  std::map<std::string, GroupState> groups_;                        // ordered: canonical table order
  std::vector<std::pair<std::string, int64_t>> pending_deny_;       // AddToDenyCache before the first round
  std::vector<std::pair<std::string, int64_t>> pending_permitted_;  // AddPermitted before the first round
  std::unordered_map<uint64_t, std::string> uid_of_id_;             // 64-bit id -> uid of every pod that reached Permit
  std::vector<std::string> node_names_;                             // snapshot index -> node name
  std::mutex mu_;                                                   // guards the maps against concurrent Less / Permit
  // last round
  PackedSnapshot packed_;
  StrIndex pod_row_;                                                // uid -> pending index
  StrIndex node_row_;                                               // node name -> snapshot index
  std::vector<std::string> group_names_;                            // table index -> "ns/name"
  std::unordered_map<std::string, uint32_t> group_row_;             // "ns/name" -> table index
  std::vector<uint8_t> prefilter_, admit_, new_denied_;
  std::vector<uint32_t> order_, rank_, feasible_;
  std::vector<int32_t> best_node_;
  std::vector<int32_t> topk_node_;                                  // [P][topk_] (BS_OUT_TOPK)
  std::vector<int64_t> topk_score_;
  std::vector<uint32_t> reasons_;                                   // [P][4 + lanes] (BS_OUT_REASONS)
  std::vector<uint32_t> ipf_reasons_;                               // [P][3] companion rows (BS_OUT_REASONS)
  std::vector<uint32_t> hp_reasons_;                                // [P] host-port companion (BS_OUT_REASONS)
  std::vector<int32_t> prio_node_;                                  // [P][priority_k_] (BS_OUT_PRIORITY)
  std::vector<int64_t> prio_score_;
  int64_t now_ns_ = 0;
  double last_pack_ms_ = 0, last_device_ms_ = 0;
  Status Reevaluate();   // bs_evaluate into the round's result vectors + the deny side effect (core.go:142,163)
  int FetchTopK();       // the round's top-K lists into topk_node_ / topk_score_ (no-op without topk)
  int FetchReasons();    // the round's reason rows into reasons_ (no-op without BS_OUT_REASONS)
  int PushRatio();      // the ratio setting with this round's lane mapping (bs_set_ratio_priority)
  int FetchPriority();   // the round's priority lists into prio_node_ / prio_score_ (no-op without priority_k)
  Status UploadNonZero(const std::vector<const Pod*>* pending);   // node column of snapshot_ (+ the pods'); no-op without
                                                                  // priority_k
  Status UploadPreferences();   // both preference sides of snapshot_ and pending_ and the two weights; the columns only
                                // while a weight is non-zero; no-op without priority_k
  Status UploadSpread();     // both spread sides of snapshot_ and pending_ and the weight; the columns only while the
                             // weight is non-zero; no-op without priority_k
  Status UploadInterPodAffinity();   // both inter-pod sides of snapshot_ and pending_ and the weight; the columns
                                    // only while the weight is non-zero; no-op without priority_k
  Status UploadInterPodFilter();   // the filter switch and, while it is on, both filter sides of snapshot_ and pending_
  Status UploadHostPorts();        // likewise for the PodFitsHostPorts filter
  Status UploadBoundHostPorts();   // the bound pods' host-port masks while the filter is on in preemption
  Status UploadLocality();   // both locality sides of snapshot_ and pending_ and the two weights; the columns only
                             // while a weight is non-zero; no-op without priority_k
  Status UploadBound();  // packs and uploads the bound-pod table of snapshot_ (no-op when no NodeInfo lists pods)
  // bs_preempt on `rows`, or with walk_flags >= 0 bs_preempt_walk with those flags
  Status RunPreempt(const std::vector<uint32_t>& rows, std::vector<Preemption>* out, int walk_flags = -1);
  std::vector<const NodeInfo*> snapshot_;                           // the round's NodeInfos (bound pods)
  std::vector<std::string> pending_uid_;                            // pending index -> uid
  std::vector<const Pod*> pending_;                                 // the round's pending pods (preferences)
  PackedBound bound_;
  StrIndex bound_row_;                                              // uid -> bound-table row
};

}  // namespace bsched
