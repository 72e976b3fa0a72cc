// plugin.cpp — snapshot packer + BatchSchedulingPlugin mirror (see plugin.hpp).
#include "plugin.hpp"

#include <omp.h>

#include <algorithm>
#include <atomic>
#include <sched.h>
#include <thread>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <set>
#include <tuple>

namespace bsched {

namespace {

constexpr int64_t kSecond = 1000000000ll;
constexpr int kLaneCpu = 0, kLaneMem = 1, kLaneEph = 2, kLanePods = 3;

double now_ms() {
  return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

bool has_prefix(const std::string& s, const char* p) { return s.rfind(p, 0) == 0; }

__int128 ipow(__int128 b, int e) {
  __int128 r = 1;
  while (e-- > 0) r *= b;
  return r;
}

}  // namespace

// resource.Quantity textual form: [sign]digits[.digits][suffix]; suffix in
//   binarySI   Ki Mi Gi Ti Pi Ei
//   decimalSI  n u m "" k M G T P E
//   exponent   e<int> | E<int>
// (k8s.io/apimachinery v0.17.5 pkg/api/resource/quantity.go, restated: source absent).
bool ParseQuantityMilli(const std::string& s, __int128* milli) {
  size_t i = 0;
  bool neg = false;
  if (i < s.size() && (s[i] == '+' || s[i] == '-')) neg = s[i++] == '-';
  __int128 mant = 0;
  int frac_digits = 0, digits = 0;
  while (i < s.size() && s[i] >= '0' && s[i] <= '9') { mant = mant * 10 + (s[i++] - '0'); if (++digits > 30) return false; }
  if (i < s.size() && s[i] == '.') {
    ++i;
    while (i < s.size() && s[i] >= '0' && s[i] <= '9') {
      mant = mant * 10 + (s[i++] - '0');
      ++frac_digits;
      if (++digits > 30) return false;
    }
  }
  if (digits == 0) return false;
  const std::string suf = s.substr(i);
  __int128 num = 1, den = 1;
  if (suf.empty()) {
  } else if (suf == "Ki") num = (__int128)1 << 10;
  else if (suf == "Mi") num = (__int128)1 << 20;
  else if (suf == "Gi") num = (__int128)1 << 30;
  else if (suf == "Ti") num = (__int128)1 << 40;
  else if (suf == "Pi") num = (__int128)1 << 50;
  else if (suf == "Ei") num = (__int128)1 << 60;
  else if (suf == "n") den = 1000000000;
  else if (suf == "u") den = 1000000;
  else if (suf == "m") den = 1000;
  else if (suf == "k") num = 1000;
  else if (suf == "M") num = 1000000;
  else if (suf == "G") num = 1000000000;
  else if (suf == "T") num = ipow(10, 12);
  else if (suf == "P") num = ipow(10, 15);
  else if (suf == "E") num = ipow(10, 18);
  else if ((suf[0] == 'e' || suf[0] == 'E') && suf.size() > 1) {
    size_t j = 1;
    bool eneg = false;
    if (suf[j] == '+' || suf[j] == '-') eneg = suf[j++] == '-';
    if (j >= suf.size()) return false;
    int ex = 0;
    for (; j < suf.size(); ++j) {
      if (suf[j] < '0' || suf[j] > '9') return false;
      ex = ex * 10 + (suf[j] - '0');
      if (ex > 24) return false;
    }
    if (eneg) den = ipow(10, ex); else num = ipow(10, ex);
  } else {
    return false;
  }
  den *= ipow(10, frac_digits);
  const __int128 n = mant * num * 1000;
  __int128 q = n / den;
  if (n % den != 0) q += 1;  // Quantity rounds up (away from zero)
  *milli = neg ? -q : q;
  return true;
}

bool QuantityMilliValue(const std::string& s, int64_t* out) {
  __int128 m;
  if (!ParseQuantityMilli(s, &m)) return false;
  if (m > (__int128)INT64_MAX || m < (__int128)INT64_MIN) return false;
  *out = (int64_t)m;
  return true;
}

bool QuantityValue(const std::string& s, int64_t* out) {
  __int128 m;
  if (!ParseQuantityMilli(s, &m)) return false;
  const bool neg = m < 0;
  __int128 a = neg ? -m : m;
  __int128 v = a / 1000 + (a % 1000 != 0 ? 1 : 0);
  if (v > (__int128)INT64_MAX) return false;
  *out = neg ? -(int64_t)v : (int64_t)v;
  return true;
}

// v1helper.IsScalarResourceName (k8s v1.17.5, restated): extended || hugepages- || prefixed native
// ("kubernetes.io/") || attachable-volumes-.  Extended: not native (has a '/', no "kubernetes.io/")
// and not prefixed "requests.".
bool IsScalarResourceName(const std::string& name) {
  if (has_prefix(name, "hugepages-") || has_prefix(name, "attachable-volumes-")) return true;
  if (name.find("kubernetes.io/") != std::string::npos) return true;
  const bool native = name.find('/') == std::string::npos;
  if (!native && !has_prefix(name, "requests.")) return true;
  return false;
}

namespace {
// labels.Requirement.Matches / NodeSelectorRequirementsAsSelector (k8s v1.17.5 apimachinery labels/selector.go,
// api/core/v1/helper, restated): valid = false when the requirement itself is malformed (the term then fails)
bool requirement_matches(const NodeSelectorRequirement& r, const std::map<std::string, std::string>& labels, bool* valid) {
  *valid = true;
  auto it = labels.find(r.key);
  const bool has = it != labels.end();
  auto in_values = [&]() {
    for (auto& v : r.values) if (v == it->second) return true;
    return false;
  };
  if (r.op == "In") {
    if (r.values.empty()) { *valid = false; return false; }
    return has && in_values();
  }
  if (r.op == "NotIn") {
    if (r.values.empty()) { *valid = false; return false; }
    return !has || !in_values();
  }
  if (r.op == "Exists") { if (!r.values.empty()) { *valid = false; return false; } return has; }
  if (r.op == "DoesNotExist") { if (!r.values.empty()) { *valid = false; return false; } return !has; }
  if (r.op == "Gt" || r.op == "Lt") {
    if (r.values.size() != 1) { *valid = false; return false; }
    char* end = nullptr;
    const long long rv = strtoll(r.values[0].c_str(), &end, 10);
    if (r.values[0].empty() || *end) { *valid = false; return false; }
    if (!has) return false;
    const long long lv = strtoll(it->second.c_str(), &end, 10);
    if (it->second.empty() || *end) return false;       // label value is not an integer: no match
    return r.op == "Gt" ? lv > rv : lv < rv;
  }
  *valid = false;
  return false;
}
// NodeSelectorRequirementsAsFieldSelector: only metadata.name with In / NotIn and exactly one value
bool field_requirement_matches(const NodeSelectorRequirement& r, const std::string& node_name, bool* valid) {
  *valid = r.key == "metadata.name" && r.values.size() == 1 && (r.op == "In" || r.op == "NotIn");
  if (!*valid) return false;
  return r.op == "In" ? node_name == r.values[0] : node_name != r.values[0];
}
}  // namespace

bool MatchNodeSelectorTerms(const std::vector<NodeSelectorTerm>& terms, const std::map<std::string, std::string>& labels,
                            const std::string& node_name) {
  for (auto& t : terms) {
    if (t.match_expressions.empty() && t.match_fields.empty()) continue;   // matches no objects
    bool ok = true, valid = true;
    for (auto& r : t.match_expressions) {
      ok = requirement_matches(r, labels, &valid) && valid;
      if (!ok) break;
    }
    if (!ok) continue;
    for (auto& r : t.match_fields) {
      ok = field_requirement_matches(r, node_name, &valid) && valid;
      if (!ok) break;
    }
    if (ok) return true;
  }
  return false;
}

bs_node_table PackedSnapshot::node_table() const {
  bs_node_table t{};
  t.n_nodes = n_nodes; t.n_lanes = lanes;
  t.alloc = alloc.data(); t.requested = requested.data(); t.pod_count = pod_count.data();
  t.alloc_present = alloc_present.data(); t.req_present = req_present.data();
  t.label_mask = label_mask.data(); t.taint_mask = taint_mask.data(); t.flags = node_flags.data();
  return t;
}
bs_pod_table PackedSnapshot::pod_table() const {
  bs_pod_table t{};
  t.n_pods = n_pods; t.n_lanes = lanes;
  t.req = req.data(); t.req_present = pod_req_present.data(); t.gid = gid.data();
  t.sel_mask = sel_mask.data(); t.tol_mask = tol_mask.data(); t.priority = priority.data();
  t.ts_ns = ts_ns.data(); t.flags = pod_flags.data();
  t.aff_class = aff_class.size() == n_pods && n_pods ? aff_class.data() : nullptr;
  return t;
}
bs_group_table PackedSnapshot::group_table() const {
  bs_group_table t{};
  t.n_groups = n_groups; t.n_lanes = lanes;
  t.min_member = min_member.data(); t.scheduled = scheduled.data(); t.matched = matched.data();
  t.flags = group_flags.data(); t.min_res = min_res.data(); t.min_res_present = min_res_present.data();
  t.rep_sel = rep_sel.data(); t.rep_tol = rep_tol.data(); t.creation_ns = creation_ns.data();
  t.name_rank = name_rank.data();
  t.rep_aff_class = rep_aff.size() == n_groups && n_groups ? rep_aff.data() : nullptr;
  return t;
}

namespace {

// What encoding one row gave, in the order a caller must see them: the std::min of two results is the one to report.
// kNeedsFull: the row holds a name the round's dictionaries have no lane or bit for (in a full pack, which built its
// dictionaries from every row, an internal error).
enum Encoded { kNeedsFull, kBadRequested, kBadAllocatable, kBadMinResources, kBadContainers, kEncoded };
const char* const kEncodeError[] = {"a row outside the round's own dictionaries", "bad quantity in requested",
                                    "bad quantity in allocatable", "bad quantity in MinResources",
                                    "bad quantity in a pod's containers"};

constexpr int kLaneIgnored = -1, kLaneUnknown = -2;

struct LaneTable {
  std::vector<std::string> scalars;
  std::unordered_map<std::string, uint32_t> lane_of;
  bool add(const std::string& scalar) {   // false: the lanes are used up
    if (lane_of.count(scalar)) return true;
    if (BS_FIXED_LANES + scalars.size() >= BS_MAX_LANES) return false;
    lane_of.emplace(scalar, BS_FIXED_LANES + (uint32_t)scalars.size());
    scalars.push_back(scalar);
    return true;
  }
  int lane(const std::string& name) const {   // kLaneUnknown: a scalar resource without a lane
    if (name == "cpu") return kLaneCpu;
    if (name == "memory") return kLaneMem;
    if (name == "ephemeral-storage") return kLaneEph;
    if (name == "pods") return kLanePods;
    if (!IsScalarResourceName(name)) return kLaneIgnored;  // Resource.Add ignores it
    auto it = lane_of.find(name);
    return it == lane_of.end() ? kLaneUnknown : (int)it->second;
  }
};

// nodeinfo.Resource.Add(rl): v[lane] += quantity (cpu in milli), scalar keys become present.  A scalar without a lane
// gives kNeedsFull even after a malformed quantity (which gives `bad`): a full pack would have given it a lane.
Encoded add_list(const LaneTable& lt, const ResourceList& rl, int64_t* v, uint32_t* present, Encoded bad) {
  Encoded r = kEncoded;
  for (auto& kv : rl) {
    const int l = lt.lane(kv.first);
    if (l == kLaneUnknown) return kNeedsFull;
    if (l < 0) continue;
    int64_t q;
    if (l == kLaneCpu ? !QuantityMilliValue(kv.second, &q) : !QuantityValue(kv.second, &q)) { r = bad; continue; }
    v[l] += q;
    if (l >= (int)BS_FIXED_LANES) *present |= 1u << l;
  }
  return r;
}

const ResourceList& container_demand(const Container& c) { return c.has_limits ? c.limits : c.requests; }  // core.go:765-769

// toleration.ToleratesTaint (k8s v1.17.5 api/core/v1/toleration.go, restated)
bool tolerates(const Toleration& t, const Taint& taint) {
  if (!t.effect.empty() && t.effect != taint.effect) return false;
  if (!t.key.empty() && t.key != taint.key) return false;
  if (t.op.empty() || t.op == "Equal") return t.value == taint.value;
  if (t.op == "Exists") return true;
  return false;
}

bool hard_taint(const Taint& t) { return t.effect == "NoSchedule" || t.effect == "NoExecute"; }  // PodToleratesNodeTaints
bool same_taint(const Taint& a, const Taint& b) { return a.key == b.key && a.value == b.value && a.effect == b.effect; }

// threads for the packer: BS_HOST_THREADS, else up to 8 (small inputs stay single-threaded)
int pack_threads(size_t objects) {
  if (objects < 4096) return 1;
  if (const char* s = getenv("BS_HOST_THREADS")) return std::max(1, atoi(s));
  int hw = (int)std::thread::hardware_concurrency();
  cpu_set_t set;   // cores this process may run on, not the box's total
  if (sched_getaffinity(0, sizeof(set), &set) == 0 && CPU_COUNT(&set) > 0) hw = std::min(hw > 0 ? hw : 1 << 20, CPU_COUNT(&set));
  return std::max(1, std::min(8, hw));
}

std::string joined_sorted(std::vector<std::string> v) {
  std::sort(v.begin(), v.end());  // sortkeys.Strings (core.go:498,507)
  std::string s;
  for (size_t i = 0; i < v.size(); ++i) { if (i) s += ","; s += v[i]; }
  return s;
}

// canonical text of a pod's node predicate beyond the selector bits ("" = none)
std::string aff_signature(const Pod& p, bool sel_in_table) {
  const bool sel = sel_in_table && !p.node_selector.empty();
  if (!p.has_required_affinity && !sel) return std::string();
  std::string s;
  if (sel)
    for (auto& kv : p.node_selector) { s += 'S'; s += kv.first; s += '\x1f'; s += kv.second; s += '\x1e'; }
  if (p.has_required_affinity) {
    s += 'A';
    for (auto& t : p.required_affinity) {
      s += 'T';
      auto put = [&](char tag, const std::vector<NodeSelectorRequirement>& rs) {
        for (auto& r : rs) {
          s += tag; s += r.key; s += '\x1f'; s += r.op; s += '\x1f';
          for (auto& v : r.values) { s += v; s += '\x1d'; }
          s += '\x1e';
        }
      };
      put('E', t.match_expressions);
      put('F', t.match_fields);
    }
  }
  return s;
}

bool aff_class_matches(const PackedSnapshot::AffClassDef& c, const Node& nd) {
  for (auto& kv : c.node_selector) {
    auto it = nd.labels.find(kv.first);
    if (it == nd.labels.end() || it->second != kv.second) return false;
  }
  return !c.has_required_affinity || MatchNodeSelectorTerms(c.terms, nd.labels, nd.name);
}

// The row encoding of one round, from the dictionaries a full pack keeps in its PackedSnapshot (scalar_names,
// sel_pairs, taint_list, sel_in_table, aff_signatures).  The full pack and the row re-packs both encode through it,
// so a re-packed row carries exactly the bits the full pack gives the same object.  The constructor sizes the node
// and group columns of `out` for out.n_nodes / out.n_groups rows, at the values of a row or field the methods leave
// out; the methods write the columns at (row, lane stride) and change nothing else, so rows may be encoded from
// several threads at once.
class RowEncoder {
 public:
  RowEncoder(const PackedSnapshot& dict, PackedSnapshot& out) : dict_(dict), out_(out) {
    for (auto& nm : dict.scalar_names) lanes_.add(nm);
    for (size_t b = 0; b < dict.sel_pairs.size(); ++b) sel_bit_.emplace(dict.sel_pairs[b], (int)b);
    for (size_t c = 0; c < dict.aff_signatures.size(); ++c) aff_class_.emplace(dict.aff_signatures[c], (uint32_t)c);
    const size_t L = dict.lanes, N = out.n_nodes, G = out.n_groups;
    out.alloc.assign(L * N, 0); out.requested.assign(L * N, 0);
    out.pod_count.assign(N, 0); out.alloc_present.assign(N, 0); out.req_present.assign(N, 0);
    out.label_mask.assign(N, 0); out.taint_mask.assign(N, 0); out.node_flags.assign(N, 0);
    out.min_member.assign(G, 0); out.scheduled.assign(G, 0); out.matched.assign(G, 0); out.group_flags.assign(G, 0);
    out.min_res.assign(L * G, 0); out.min_res_present.assign(G, 0); out.rep_sel.assign(G, 0);
    out.rep_tol.assign(G, 0); out.creation_ns.assign(G, 0); out.name_rank.assign(G, 0); out.wait_ns.assign(G, 0);
    out.rep_aff.assign(G, BS_AFF_NONE);
  }

  Encoded node(const NodeInfo* ni, uint32_t i, uint32_t stride) const {
    if (!ni) { out_.node_flags[i] = BS_NODE_NIL; return kEncoded; }                   // core.go:606
    const Node* nd = ni->node;
    int64_t req[BS_MAX_LANES] = {}, alloc[BS_MAX_LANES] = {};
    uint32_t req_pres = 0, alloc_pres = 0;
    const Encoded r = std::min(add_list(lanes_, ni->requested, req, &req_pres, kBadRequested),
                               nd ? add_list(lanes_, nd->allocatable, alloc, &alloc_pres, kBadAllocatable) : kEncoded);
    if (r != kEncoded) return r;
    uint8_t fl = 0;
    if (!nd) fl |= BS_NODE_NO_NODE;                                                    // core.go:610
    if (ni->taints_error) fl |= BS_NODE_TAINTS_ERR;                                    // core.go:639
    if (nd && nd->unschedulable) fl |= BS_NODE_UNSCHEDULABLE;                          // core.go:615
    out_.node_flags[i] = fl;
    out_.pod_count[i] = ni->num_pods;
    for (uint32_t d = 0; d < dict_.lanes; ++d) {
      out_.requested[(size_t)d * stride + i] = req[d];
      out_.alloc[(size_t)d * stride + i] = alloc[d];
    }
    out_.req_present[i] = req_pres;
    out_.alloc_present[i] = alloc_pres;
    if (!nd) return kEncoded;
    for (size_t b = 0; b < dict_.sel_pairs.size(); ++b) {
      auto it = nd->labels.find(dict_.sel_pairs[b].first);
      if (it != nd->labels.end() && it->second == dict_.sel_pairs[b].second) out_.label_mask[i] |= 1ull << b;
    }
    for (auto& t : nd->taints) {
      if (!hard_taint(t)) continue;
      const int b = taint_bit(t);
      if (b < 0) return kNeedsFull;   // a taint no toleration mask of the round has a bit for
      out_.taint_mask[i] |= 1ull << b;
    }
    return kEncoded;
  }

  // everything of a group's row but name_rank, which depends on the other groups' names
  Encoded group(const BatchSchedulingPlugin::GroupDelta& gd, uint32_t k, uint32_t stride, int64_t default_wait_ns) const {
    const PodGroup& pg = *gd.pg;
    out_.min_member[k] = pg.min_member;
    out_.scheduled[k] = pg.scheduled;
    out_.matched[k] = gd.matched;
    out_.creation_ns[k] = pg.creation_ns;
    // util.GetWaitTimeDuration (k8s.go:82-91): Spec.MaxScheduleTime wins, else the plugin default
    out_.wait_ns[k] = pg.max_schedule_time_ns >= 0 ? pg.max_schedule_time_ns : default_wait_ns;
    uint8_t fl = gd.flags & (BS_GROUP_SCHEDULED | BS_GROUP_HAS_POD | BS_GROUP_DENIED);
    if (pg.has_min_resources) {
      fl |= BS_GROUP_HAS_MINRES;
      int64_t v[BS_MAX_LANES] = {};
      uint32_t pres = 0;
      const Encoded r = add_list(lanes_, pg.min_resources, v, &pres, kBadMinResources);
      if (r != kEncoded) return r;
      for (uint32_t d = 0; d < dict_.lanes; ++d) out_.min_res[(size_t)d * stride + k] = v[d];
      out_.min_res_present[k] = pres;
    }
    if (gd.rep_pod) {
      fl |= BS_GROUP_HAS_POD;
      const std::string sig = aff_signature(*gd.rep_pod, dict_.sel_in_table);
      if (!sig.empty()) {
        auto it = aff_class_.find(sig);
        if (it == aff_class_.end()) return kNeedsFull;   // a predicate the round's table has no row for
        out_.rep_aff[k] = it->second;
      }
      const Encoded r = pod_masks(*gd.rep_pod, &out_.rep_sel[k], &out_.rep_tol[k]);
      if (r != kEncoded) return r;
    }
    out_.group_flags[k] = fl;
    return kEncoded;
  }

  // nodeSelector pairs -> selector bits (none while the selectors live in the affinity table), tolerations -> the
  // bits of the taints they tolerate
  Encoded pod_masks(const Pod& p, uint64_t* sel, uint64_t* tol) const {
    *sel = 0;
    *tol = 0;
    if (!dict_.sel_in_table)
      for (auto& kv : p.node_selector) {
        auto it = sel_bit_.find(kv);
        if (it == sel_bit_.end()) return kNeedsFull;   // the nodes' label masks have no bit for this pair
        *sel |= 1ull << it->second;
      }
    for (size_t b = 0; b < dict_.taint_list.size(); ++b)
      for (auto& tl : p.tolerations)
        if (tolerates(tl, dict_.taint_list[b])) { *tol |= 1ull << b; break; }
    return kEncoded;
  }

 private:
  int taint_bit(const Taint& t) const {
    for (size_t b = 0; b < dict_.taint_list.size(); ++b)
      if (same_taint(dict_.taint_list[b], t)) return (int)b;
    return -1;
  }

  const PackedSnapshot& dict_;
  PackedSnapshot& out_;
  LaneTable lanes_;
  std::map<std::pair<std::string, std::string>, int> sel_bit_;
  std::unordered_map<std::string, uint32_t> aff_class_;
};

Status pack_impl(const std::vector<const NodeInfo*>& snapshot, const std::vector<const Pod*>& pending,
                 const std::vector<BatchSchedulingPlugin::GroupDelta>& groups, const std::vector<uint8_t>& pod_flags_in,
                 int64_t default_wait_ns, PackedSnapshot* out) {
  Status bad{BS_CODE_ERROR, ""};
  PackedSnapshot& ps = *out;
  ps = PackedSnapshot();
  const uint32_t N = (uint32_t)snapshot.size(), P = (uint32_t)pending.size(), G = (uint32_t)groups.size();
  const bool prof = getenv("BS_PACK_PROFILE") != nullptr;
  double tp = now_ms();
  auto phase = [&](const char* name) {
    if (!prof) return;
    const double t = now_ms();
    fprintf(stderr, "[pack] %-12s %.2f ms\n", name, t - tp);
    tp = t;
  };
  // ---- lanes: scalar resources in first-seen order (nodes, groups, pods)
  // Objects are scanned in parallel; each thread records the scalar names it meets with the position
  // (object class, index) of their first appearance, and the merge keeps the global first-seen order.
  LaneTable lt;
  const int T = pack_threads((size_t)N + P + G);
  {
    struct Seen { uint64_t pos; std::string name; };
    std::vector<std::vector<Seen>> seen(T);
    auto note = [&](std::vector<Seen>& mine, uint64_t pos, const ResourceList& rl) {
      for (auto& kv : rl) {
        const std::string& nm = kv.first;
        if (lt.lane(nm) != kLaneUnknown) continue;   // lt stays empty until the merge: only the scalars are noted
        bool dup = false;
        for (auto& s2 : mine) if (s2.name == nm) { dup = true; break; }
        if (!dup) mine.push_back(Seen{pos, nm});
      }
    };
#pragma omp parallel num_threads(T)
    {
      std::vector<Seen>& mine = seen[omp_get_thread_num()];
#pragma omp for schedule(static) nowait
      for (uint32_t i = 0; i < N; ++i) {
        const NodeInfo* ni = snapshot[i];
        if (!ni) continue;
        if (ni->node) note(mine, ((uint64_t)0 << 40) | ((uint64_t)i << 1), ni->node->allocatable);
        note(mine, ((uint64_t)0 << 40) | ((uint64_t)i << 1) | 1, ni->requested);
      }
#pragma omp for schedule(static) nowait
      for (uint32_t g = 0; g < G; ++g)
        if (groups[g].pg->has_min_resources) note(mine, ((uint64_t)1 << 40) | g, groups[g].pg->min_resources);
#pragma omp for schedule(static) nowait
      for (uint32_t i = 0; i < P; ++i)
        for (auto& c : pending[i]->containers) note(mine, ((uint64_t)2 << 40) | i, container_demand(c));
#pragma omp for schedule(static) nowait
      for (uint32_t g = 0; g < G; ++g)
        if (groups[g].rep_pod)
          for (auto& c : groups[g].rep_pod->containers) note(mine, ((uint64_t)3 << 40) | g, container_demand(c));
    }
    std::vector<Seen> all;
    for (auto& v : seen) all.insert(all.end(), v.begin(), v.end());
    std::stable_sort(all.begin(), all.end(), [](const Seen& a, const Seen& b) { return a.pos < b.pos; });
    for (auto& s2 : all)
      if (!lt.add(s2.name)) { bad.message = "more than 12 scalar resources"; return bad; }
  }
  phase("lane scan");
  const uint32_t L = BS_FIXED_LANES + (uint32_t)lt.scalars.size();
  ps.lanes = L;
  ps.scalar_names = lt.scalars;
  ps.n_nodes = N; ps.n_pods = P; ps.n_groups = G;

  // ---- selector pairs and taints -> bits
  std::set<std::pair<std::string, std::string>> pairs;
  for (auto* p : pending) pairs.insert(p->node_selector.begin(), p->node_selector.end());
  for (auto& g : groups) if (g.rep_pod) pairs.insert(g.rep_pod->node_selector.begin(), g.rep_pod->node_selector.end());
  // more than 64 distinct pairs: every nodeSelector moves into the affinity table (one class per distinct
  // selector map), the 64-bit masks stay zero
  ps.sel_in_table = pairs.size() > 64;
  if (!ps.sel_in_table) ps.sel_pairs.assign(pairs.begin(), pairs.end());
  // ---- affinity classes: first-seen order over the pending pods, then the groups' representatives
  {
    std::unordered_map<std::string, uint32_t> cls;
    auto class_of = [&](const Pod& p) -> uint32_t {
      const std::string sig = aff_signature(p, ps.sel_in_table);
      if (sig.empty()) return BS_AFF_NONE;
      auto it = cls.find(sig);
      if (it != cls.end()) return it->second;
      const uint32_t id = (uint32_t)ps.aff_classes.size();
      PackedSnapshot::AffClassDef d;
      if (ps.sel_in_table) d.node_selector = p.node_selector;
      d.has_required_affinity = p.has_required_affinity;
      d.terms = p.required_affinity;
      ps.aff_classes.push_back(std::move(d));
      ps.aff_signatures.push_back(sig);
      cls.emplace(sig, id);
      return id;
    };
    ps.aff_class.assign(P, BS_AFF_NONE);
    bool any = ps.sel_in_table;
    for (uint32_t i = 0; i < P && !any; ++i) any = pending[i]->has_required_affinity;
    for (uint32_t g = 0; g < G && !any; ++g) any = groups[g].rep_pod && groups[g].rep_pod->has_required_affinity;
    if (any) {
      for (uint32_t i = 0; i < P; ++i) ps.aff_class[i] = class_of(*pending[i]);
      for (uint32_t g = 0; g < G; ++g) if (groups[g].rep_pod) class_of(*groups[g].rep_pod);   // rep_aff: RowEncoder::group
    }
  }
  phase("selectors");
  // taints: first-seen order defines the bit
  for (uint32_t i = 0; i < N; ++i) {
    const NodeInfo* ni = snapshot[i];
    if (!ni || !ni->node) continue;
    for (auto& t : ni->node->taints)
      if (hard_taint(t) && std::none_of(ps.taint_list.begin(), ps.taint_list.end(), [&](const Taint& u) { return same_taint(u, t); }))
        ps.taint_list.push_back(t);
  }
  if (ps.taint_list.size() > 64) { bad.message = "more than 64 distinct taints in one round"; return bad; }
  // ---- rows, through the encoding PackNodeRows / PackGroupRows use
  const RowEncoder enc(ps, ps);
  std::atomic<int> err{kEncoded};
  auto failed = [&] { bad.message = kEncodeError[err]; return bad; };
#pragma omp parallel for num_threads(T) schedule(static)
  for (uint32_t i = 0; i < N; ++i) {
    const Encoded r = enc.node(snapshot[i], i, N);
    if (r != kEncoded) err = r;
  }
  if (err != kEncoded) return failed();
  phase("nodes");
  // ---- (affinity class, node) verdicts, evaluated on the host once per class and node
  {
    const uint32_t A = ps.n_aff(), W = (N + 31) / 32;
    ps.aff_bits.assign((size_t)A * W, 0);
#pragma omp parallel for num_threads(T) schedule(static) collapse(2)
    for (uint32_t c = 0; c < A; ++c)
      for (uint32_t w = 0; w < W; ++w) {
        uint32_t word = 0;
        for (uint32_t b = 0; b < 32 && w * 32 + b < N; ++b) {
          const NodeInfo* ni = snapshot[w * 32 + b];
          if (ni && ni->node && aff_class_matches(ps.aff_classes[c], *ni->node)) word |= 1u << b;
        }
        ps.aff_bits[(size_t)c * W + w] = word;
      }
  }
  phase("affinity");
  auto pod_demand = [&](const Pod& p, int64_t* v, uint32_t* pres) {  // getPodResourceRequire core.go:761-772
    for (auto& c : p.containers) {
      const Encoded r = add_list(lt, container_demand(c), v, pres, kBadContainers);
      if (r != kEncoded) return r;
    }
    return kEncoded;
  };
  // ---- groups
  // bare-name ranks, byte-wise ascending (Go string compare); equal names share a rank (core.go:404)
  // (sorted on the big-endian first 8 bytes as an integer; the strings are compared only where those tie)
  std::vector<uint32_t> by_name(G);
  {
    struct NameKey { uint64_t pre; uint32_t g; };
    std::vector<NameKey> nk(G);
#pragma omp parallel for num_threads(T) schedule(static)
    for (uint32_t g = 0; g < G; ++g) {
      const std::string& nm = groups[g].pg->name;
      uint64_t pre = 0;
      for (size_t b = 0; b < 8; ++b) pre = (pre << 8) | (b < nm.size() ? (unsigned char)nm[b] : 0u);
      nk[g] = NameKey{pre, g};
    }
    std::sort(nk.begin(), nk.end(), [&](const NameKey& a, const NameKey& b) {
      if (a.pre != b.pre) return a.pre < b.pre;
      return groups[a.g].pg->name < groups[b.g].pg->name;   // equal prefixes (incl. a short name vs one with NUL bytes)
    });
    for (uint32_t k = 0; k < G; ++k) by_name[k] = nk[k].g;
  }
  std::vector<uint32_t> rank_of_group(G);
  {
    uint32_t r = 0;
    for (uint32_t k = 0; k < G; ++k) {
      if (k > 0 && groups[by_name[k]].pg->name != groups[by_name[k - 1]].pg->name) ++r;
      rank_of_group[by_name[k]] = r;
    }
  }
  // "ns/name" -> group row (the lister's key, util.GetPodGroupFullName): a flat open-addressing table over a
  // 64-bit hash of the two strings — no key is concatenated or allocated, neither here nor in the pods' lookups.
  // The first row with a given full name wins, as a map insert would.
  auto full_hash = [](const std::string& ns, const std::string& name) {
    uint64_t h = 1469598103934665603ull;
    for (unsigned char c : ns) h = (h ^ c) * 1099511628211ull;
    h = (h ^ (unsigned char)'/') * 1099511628211ull;
    for (unsigned char c : name) h = (h ^ c) * 1099511628211ull;
    return h ^ (h >> 32);
  };
  uint32_t gmask = 1;
  while (gmask < 2 * std::max(G, 1u)) gmask <<= 1;
  gmask -= 1;
  std::vector<uint32_t> gslot((size_t)gmask + 1, 0xffffffffu);
  {
    std::vector<uint64_t> gh(G);
#pragma omp parallel for num_threads(T) schedule(static)
    for (uint32_t g = 0; g < G; ++g) gh[g] = full_hash(groups[g].pg->ns, groups[g].pg->name);
    for (uint32_t g = 0; g < G; ++g) {
      uint32_t sl = (uint32_t)gh[g] & gmask;
      bool dup = false;
      while (gslot[sl] != 0xffffffffu) {
        const PodGroup& o = *groups[gslot[sl]].pg;
        if (o.name == groups[g].pg->name && o.ns == groups[g].pg->ns) { dup = true; break; }
        sl = (sl + 1) & gmask;
      }
      if (!dup) gslot[sl] = g;
    }
  }
  auto find_group = [&](const std::string& ns, const std::string& name) -> int32_t {
    uint32_t sl = (uint32_t)full_hash(ns, name) & gmask;
    while (gslot[sl] != 0xffffffffu) {
      const PodGroup& o = *groups[gslot[sl]].pg;
      if (o.name == name && o.ns == ns) return (int32_t)gslot[sl];
      sl = (sl + 1) & gmask;
    }
    return -1;
  };
#pragma omp parallel for num_threads(T) schedule(static)
  for (uint32_t g = 0; g < G; ++g) {
    ps.name_rank[g] = rank_of_group[g];
    const Encoded r = enc.group(groups[g], g, G, default_wait_ns);
    if (r != kEncoded) err = r;
  }
  if (err != kEncoded) return failed();
  phase("groups");
  // ---- pods (arrival order): demand / masks / group lookup in parallel, then the occupancy
  // rule sequentially, as fillOccupiedObj is order dependent (core.go:494-511)
  ps.req.assign((size_t)L * P, 0); ps.pod_req_present.assign(P, 0); ps.gid.assign(P, BS_GID_NONE);
  ps.sel_mask.assign(P, 0); ps.tol_mask.assign(P, 0); ps.priority.assign(P, 0); ps.ts_ns.assign(P, 0);
  ps.pod_flags.assign(P, 0);
#pragma omp parallel for num_threads(T) schedule(static)
  for (uint32_t i = 0; i < P; ++i) {
    const Pod& p = *pending[i];
    uint32_t pres = 0;
    int64_t tmp[BS_MAX_LANES] = {};
    Encoded r = pod_demand(p, tmp, &pres);
    if (r == kEncoded) r = enc.pod_masks(p, &ps.sel_mask[i], &ps.tol_mask[i]);
    if (r != kEncoded) { err = r; continue; }
    for (uint32_t d = 0; d < L; ++d) ps.req[(size_t)d * P + i] = tmp[d];
    ps.pod_req_present[i] = pres;
    ps.priority[i] = p.priority;
    ps.ts_ns[i] = p.queue_ts_ns;
    uint8_t fl = i < pod_flags_in.size() ? pod_flags_in[i] : 0;
    auto lab = p.labels.find(kPodGroupLabel);                          // util.VerifyPodLabelSatisfied k8s.go:62-70
    if (lab != p.labels.end() && !lab->second.empty()) {
      const int32_t gi = find_group(p.ns, lab->second);
      if (gi < 0) { ps.gid[i] = BS_GID_MISSING; fl |= BS_POD_LISTER_MISS; }
      else ps.gid[i] = gi;
    }
    ps.pod_flags[i] = fl;
  }
  if (err != kEncoded) return failed();
  phase("pods par");
  // fillOccupiedObj runs when a pod is popped, i.e. in QUEUE order (Less = Compare, core.go:368-411), not in
  // arrival order: with an empty OccupiedBy and pods of one group carrying different ownerRefs, the first pod
  // in queue order decides who occupies the group.  Stable sort of the grouped pods by Compare's key.
  // Only pods of one group interact, and within a group Compare's key reduces to (priority desc, timestamp asc)
  // with arrival order on ties — so the pods are bucketed by group (counting sort, arrival order kept) and every
  // group replays its own few pods in queue order, groups in parallel.
  {
    std::vector<uint32_t> start((size_t)G + 1, 0);
    for (uint32_t i = 0; i < P; ++i)
      if (ps.gid[i] >= 0) ++start[(size_t)ps.gid[i] + 1];
    for (uint32_t g = 0; g < G; ++g) start[g + 1] += start[g];
    std::vector<uint32_t> bucket(start[G]);
    {
      std::vector<uint32_t> fill(start.begin(), start.end() - 1);
      for (uint32_t i = 0; i < P; ++i)
        if (ps.gid[i] >= 0) bucket[fill[ps.gid[i]]++] = i;
    }
#pragma omp parallel for num_threads(T) schedule(dynamic, 2048)
    for (uint32_t g = 0; g < G; ++g) {
      uint32_t* b0 = bucket.data() + start[g];
      uint32_t* b1 = bucket.data() + start[g + 1];
      if (b0 == b1 || (ps.group_flags[g] & BS_GROUP_DENIED)) continue;   // a frozen group: no pod reaches fillOccupiedObj
      std::stable_sort(b0, b1, [&](uint32_t x, uint32_t y) {
        if (ps.priority[x] != ps.priority[y]) return ps.priority[x] > ps.priority[y];
        return ps.ts_ns[x] < ps.ts_ns[y];
      });
      std::string occ = groups[g].pg->occupied_by;
      for (uint32_t* q = b0; q != b1; ++q) {
        const uint32_t i = *q;
        uint8_t fl = ps.pod_flags[i];
        if (fl & BS_POD_PERMITTED_RECENTLY) continue;
        const Pod& p = *pending[i];
        if (occ.empty()) {
          if (!p.owner_uids.empty()) occ = joined_sorted(p.owner_uids);             // core.go:496-500
        } else if (p.owner_uids.empty()) fl |= BS_POD_OCC_NOREFS;                   // core.go:504-506
        else if (joined_sorted(p.owner_uids) != occ) fl |= BS_POD_OCC_MISMATCH;    // core.go:507-510
        ps.pod_flags[i] = fl;
      }
    }
  }
  phase("occupancy");
  return Status{};
}

}  // namespace

Status BatchSchedulingPlugin::Pack(const std::vector<const NodeInfo*>& snapshot, const std::vector<const Pod*>& pending,
                                   const std::vector<PodGroup>& groups, const std::vector<uint32_t>& matched,
                                   const std::vector<uint8_t>& extra_group_flags,
                                   const std::vector<uint8_t>& extra_pod_flags, int64_t default_wait_ns,
                                   PackedSnapshot* out) {
  std::vector<GroupDelta> gd(groups.size());
  for (size_t g = 0; g < groups.size(); ++g)
    gd[g] = GroupDelta{(uint32_t)g, &groups[g], g < matched.size() ? matched[g] : 0u,
                       g < extra_group_flags.size() ? extra_group_flags[g] : (uint8_t)0, nullptr};
  return Pack(snapshot, pending, gd, extra_pod_flags, default_wait_ns, out);
}

Status BatchSchedulingPlugin::Pack(const std::vector<const NodeInfo*>& snapshot, const std::vector<const Pod*>& pending,
                                   const std::vector<GroupDelta>& groups, const std::vector<uint8_t>& extra_pod_flags,
                                   int64_t default_wait_ns, PackedSnapshot* out) {
  for (auto& g : groups)
    if (!g.pg) return Status{BS_CODE_ERROR, "Pack: null PodGroup"};
  return pack_impl(snapshot, pending, groups, extra_pod_flags, default_wait_ns, out);
}

BatchSchedulingPlugin::BatchSchedulingPlugin(int device, int64_t max_schedule_time_ns, uint32_t out_flags, uint32_t topk,
                                             uint32_t priority_k)
    : max_schedule_time_ns_(max_schedule_time_ns) {
  device_ = device;
  out_flags_ = out_flags | (topk ? BS_OUT_TOPK : 0u) | (priority_k ? BS_OUT_PRIORITY : 0u);
  topk_ = topk;
  priority_k_ = priority_k;
  if (topk && priority_k && topk != priority_k) init_error_ = "topk and priority_k share one list length: they must be equal";
}

BatchSchedulingPlugin::~BatchSchedulingPlugin() {
  if (eng_) bs_destroy(eng_);
}

void BatchSchedulingPlugin::SetPodGroup(const PodGroup& pg) {
  std::lock_guard<std::mutex> lk(mu_);
  GroupState& gs = groups_[pg.ns + "/" + pg.name];
  gs.pg = pg;
}

void BatchSchedulingPlugin::DeletePodGroup(const std::string& ns_name) {
  std::lock_guard<std::mutex> lk(mu_);
  groups_.erase(ns_name);
}

uint64_t BatchSchedulingPlugin::IdOf(const std::string& s) {
  uint64_t h = 1469598103934665603ull;
  for (unsigned char c : s) { h ^= c; h *= 1099511628211ull; }
  return h;
}

void BatchSchedulingPlugin::AddToDenyCache(const std::string& ns_name, int64_t now_ns) {
  const int g = group_index(ns_name);
  if (eng_ && g >= 0) bs_deny(eng_, (uint32_t)g, now_ns);          // lastDeniedPG.Add(.., 20 s)  core.go:424 (Add: Q11)
  else pending_deny_.push_back({ns_name, now_ns});
}

void BatchSchedulingPlugin::AddPermitted(const std::string& uid, int64_t now_ns) {
  if (eng_) bs_mark_permitted(eng_, IdOf(uid), now_ns);           // core.go:188
  else pending_permitted_.push_back({uid, now_ns});
}

Status BatchSchedulingPlugin::Tick(int64_t now_ns, std::vector<std::string>* rejected_uids,
                                   std::vector<std::string>* evicted_groups) {
  if (!eng_) return Status{};
  std::lock_guard<std::mutex> lk(mu_);
  const uint32_t cap = (uint32_t)uid_of_id_.size() + 1, G = (uint32_t)group_names_.size();
  std::vector<uint32_t> rg(cap), ev(G + 1);
  std::vector<uint64_t> ru(cap);
  uint32_t nr = 0, ne = 0;
  const int rc = bs_expire(eng_, now_ns, rg.data(), ru.data(), cap, &nr, ev.data(), G + 1, &ne);
  if (rc) return Status{BS_CODE_ERROR, std::string("bsched: ") + bs_strerror(rc)};
  for (uint32_t i = 0; i < nr && i < cap; ++i) {
    auto it = uid_of_id_.find(ru[i]);
    if (rejected_uids && it != uid_of_id_.end()) rejected_uids->push_back(it->second);
  }
  for (uint32_t i = 0; i < ne && i < G + 1; ++i)
    if (evicted_groups && ev[i] < G) evicted_groups->push_back(group_names_[ev[i]]);
  return Status{};
}

Status BatchSchedulingPlugin::AllowList(const std::string& ns_name, int64_t now_ns,
                                        std::vector<std::pair<std::string, std::string>>* allow) {
  if (!eng_ || !allow) return Status{BS_CODE_ERROR, "AllowList: no round has been started"};
  std::lock_guard<std::mutex> lk(mu_);
  const int g = group_index(ns_name);
  if (g < 0) return Status{BS_CODE_ERROR, "AllowList: unknown group"};
  const uint32_t cap = (uint32_t)uid_of_id_.size() + 1;
  std::vector<uint64_t> u(cap);
  std::vector<uint32_t> nd(cap);
  uint32_t n = 0;
  const int rc = bs_allow_list(eng_, (uint32_t)g, now_ns, u.data(), nd.data(), cap, &n);
  if (rc) return Status{BS_CODE_ERROR, std::string("bsched: ") + bs_strerror(rc)};
  for (uint32_t i = 0; i < n && i < cap; ++i) {
    auto it = uid_of_id_.find(u[i]);
    allow->push_back({it != uid_of_id_.end() ? it->second : std::string(), nd[i] < node_names_.size() ? node_names_[nd[i]] : std::string()});
  }
  return Status{};
}

int BatchSchedulingPlugin::group_index(const std::string& ns_name) const {
  auto it = group_row_.find(ns_name);
  return it == group_row_.end() ? -1 : (int)it->second;
}

Status BatchSchedulingPlugin::BeginRound(const std::vector<const NodeInfo*>& snapshot,
                                         const std::vector<const Pod*>& pending, int64_t now_ns) {
  const double t0 = now_ms();
  if (!init_error_.empty()) return Status{BS_CODE_ERROR, init_error_};
  std::lock_guard<std::mutex> lk(mu_);
  now_ns_ = now_ns;
  const bool prof = getenv("BS_PACK_PROFILE") != nullptr;
  double tp = t0;
  auto lap = [&](const char* what) {
    if (!prof) return;
    const double t = now_ms();
    fprintf(stderr, "[begin] %-12s %.2f ms\n", what, t - tp);
    tp = t;
  };
  // the group table of this round (canonical order = the map's) and how it continues the last one's rows
  // (the usual cycle has the same PodGroups as the last one: one pass of string compares, nothing rebuilt)
  bool same = group_names_.size() == groups_.size();
  if (same) {
    size_t i = 0;
    for (auto& kv : groups_)
      if (kv.first != group_names_[i++]) { same = false; break; }
  }
  const uint32_t Gn = (uint32_t)groups_.size();
  if (!same) {
    std::vector<std::string> names;
    std::vector<int32_t> old_index;
    names.reserve(Gn);
    old_index.reserve(Gn);
    for (auto& kv : groups_) {
      auto it = group_row_.find(kv.first);
      old_index.push_back(it == group_row_.end() ? -1 : (int32_t)it->second);
      names.push_back(kv.first);
    }
    if (eng_ && state_ready_) {
      const int rc = bs_state_remap(eng_, Gn, old_index.data());
      if (rc) return Status{BS_CODE_ERROR, std::string("bsched: ") + bs_strerror(rc)};
    }
    group_names_.swap(names);
    group_row_.clear();
    group_row_.reserve(Gn);
    for (uint32_t g = 0; g < Gn; ++g) group_row_[group_names_[g]] = g;
  }
  lap("group names");
  // the engine's TTL tables as of now: matched counts, pgs.Scheduled, deny list, recently permitted uids
  std::vector<uint32_t> st_matched(Gn, 0);
  std::vector<uint8_t> st_flags(Gn, 0);
  if (eng_ && state_ready_ && Gn) {
    const int rc = bs_state_view(eng_, now_ns, Gn, st_matched.data(), st_flags.data());
    if (rc) return Status{BS_CODE_ERROR, std::string("bsched: ") + bs_strerror(rc)};
  }
  std::vector<GroupDelta> gin;
  gin.reserve(Gn);
  {
    uint32_t g = 0;
    for (auto& kv : groups_) {
      GroupState& gs = kv.second;
      gin.push_back(GroupDelta{g, &gs.pg, st_matched[g], st_flags[g], gs.has_pod ? &gs.rep_pod : nullptr});
      ++g;
    }
  }
  lap("group rows");
  std::vector<uint8_t> pflags(pending.size(), 0);
  std::vector<uint64_t> uid_ids(pending.size()), name_ids(pending.size());
  const int T = pack_threads(pending.size());
  pod_row_.build(pending.size(), [&](size_t i) { return &pending[i]->uid; }, T);
  {
    // ids of the uids and of "ns/name" (FNV-1a streams: hashing ns, '/', name in turn equals hashing the joined string)
#pragma omp parallel for num_threads(T) schedule(static)
    for (size_t i = 0; i < pending.size(); ++i) {
      uid_ids[i] = IdOf(pending[i]->uid);
      uint64_t h = 1469598103934665603ull;
      for (unsigned char c : pending[i]->ns) { h ^= c; h *= 1099511628211ull; }
      h ^= (unsigned char)'/'; h *= 1099511628211ull;
      for (unsigned char c : pending[i]->name) { h ^= c; h *= 1099511628211ull; }
      name_ids[i] = h;
    }
  }
  lap("pod rows+ids");
  if (eng_ && state_ready_ && !pending.empty()) {
    std::vector<uint8_t> perm(pending.size());
    bs_permitted_view(eng_, now_ns, uid_ids.data(), (uint32_t)pending.size(), perm.data());
    for (size_t i = 0; i < pending.size(); ++i)
      if (perm[i]) pflags[i] |= BS_POD_PERMITTED_RECENTLY;
  }
  node_row_.build(snapshot.size(), [&](size_t i) { return snapshot[i] && snapshot[i]->node ? &snapshot[i]->node->name : nullptr; },
                  pack_threads(snapshot.size()));
  node_names_.assign(snapshot.size(), std::string());
  snapshot_ = snapshot;
  pending_uid_.resize(pending.size());
  pending_ = pending;
  for (size_t i = 0; i < pending.size(); ++i) pending_uid_[i] = pending[i]->uid;
  for (size_t i = 0; i < snapshot.size(); ++i)
    if (snapshot[i] && snapshot[i]->node) node_names_[i] = snapshot[i]->node->name;
  lap("node rows");
  Status st = pack_impl(snapshot, pending, gin, pflags, max_schedule_time_ns_, &packed_);
  if (!st.ok()) return st;
  lap("pack_impl");
  last_pack_ms_ = now_ms() - t0;

  const double t1 = now_ms();
  auto fail = [&](int rc) {
    Status s{BS_CODE_ERROR, std::string("bsched: ") + bs_strerror(rc)};
    if (eng_) s.message += std::string(" (") + bs_last_error(eng_) + ")";
    return s;
  };
  if (!eng_ || eng_lanes_ != packed_.lanes) {
    // a new scalar resource changed the lane count: a fresh engine takes over the gang state of the old one
    bs_engine* fresh = nullptr;
    bs_config cfg{device_, packed_.lanes, out_flags_, topk_ ? topk_ : priority_k_};
    int rc = bs_create(&cfg, &fresh);
    if (rc) return fail(rc);
    if (eng_) { bs_state_move(fresh, eng_); bs_destroy(eng_); }
    eng_ = fresh;
    eng_lanes_ = packed_.lanes;
  }
  bs_node_table nt = packed_.node_table();
  bs_group_table gt = packed_.group_table();
  bs_pod_table pt = packed_.pod_table();
  int rc;
  if ((rc = bs_upload_nodes(eng_, &nt))) return fail(rc);
  if (packed_.n_aff() && (rc = bs_upload_affinity(eng_, packed_.n_aff(), packed_.aff_bits.data()))) return fail(rc);
  if ((rc = bs_upload_groups(eng_, &gt))) return fail(rc);
  if ((rc = bs_upload_pods(eng_, &pt))) return fail(rc);
  {
    Status nst = UploadNonZero(&pending);
    if (!nst.ok()) return nst;
    nst = UploadPreferences();
    if (!nst.ok()) return nst;
    nst = UploadLocality();
    if (!nst.ok()) return nst;
    nst = UploadSpread();
    if (!nst.ok()) return nst;
    nst = UploadInterPodAffinity();
    if (!nst.ok()) return nst;
    nst = UploadInterPodFilter();
    if (!nst.ok()) return nst;
    nst = UploadHostPorts();
    if (!nst.ok()) return nst;
  }
  {
    Status bst = UploadBound();   // after the groups: the bound rows' group indices refer to this table
    if (!bst.ok()) return bst;
  }
  if ((rc = bs_set_wait_time(eng_, max_schedule_time_ns_, packed_.wait_ns.data(), packed_.n_groups))) return fail(rc);
  if (!state_ready_) {
    if ((rc = bs_state_reset(eng_))) return fail(rc);
    state_ready_ = true;
  }
  for (auto& d : pending_deny_) { const int g = group_index(d.first); if (g >= 0) bs_deny(eng_, (uint32_t)g, d.second); }
  for (auto& d : pending_permitted_) bs_mark_permitted(eng_, IdOf(d.first), d.second);
  pending_deny_.clear();
  pending_permitted_.clear();
  if ((rc = bs_set_pod_ids(eng_, uid_ids.data(), name_ids.data()))) return fail(rc);
  if ((rc = bs_begin_cycle(eng_, now_ns))) return fail(rc);   // the round reads the engine's own tables
  const uint32_t P = packed_.n_pods, G = packed_.n_groups;
  prefilter_.assign(P, 0); feasible_.assign(P, 0); best_node_.assign(P, -1); order_.assign(P, 0); rank_.assign(P, 0);
  admit_.assign(G, 0); new_denied_.assign(G, 0);
  bs_results r{};
  r.prefilter = prefilter_.data(); r.feasible_count = feasible_.data(); r.best_node = best_node_.data();
  r.admit = admit_.data(); r.new_denied = new_denied_.data(); r.order = order_.data(); r.rank = rank_.data();
  if ((rc = bs_evaluate(eng_, &r))) return fail(rc);
  if ((rc = FetchTopK())) return fail(rc);
  if ((rc = FetchReasons())) return fail(rc);
  if ((rc = FetchPriority())) return fail(rc);
  last_device_ms_ = now_ms() - t1;

  // side effects the reference performs while it walks the pods:
  //  * AddToDenyCache for every group refused with "cluster resource not enough" (core.go:142,163)
  //  * fillOccupiedObj: first reaching pod becomes pgs.Pod, supplies MinResources / OccupiedBy
  // (AddToDenyCache for the groups refused with "cluster resource not enough", core.go:142,163, happened inside
  //  the engine when the round was fetched)
  for (uint32_t i = 0; i < P; ++i) {
    const int32_t g = packed_.gid[i];
    if (g < 0) continue;
    if (packed_.pod_flags[i] & BS_POD_PERMITTED_RECENTLY) continue;
    if (packed_.group_flags[g] & BS_GROUP_DENIED) continue;
    GroupState& gs = groups_[group_names_[g]];
    const Pod& p = *pending[i];
    if (!gs.has_pod) { gs.has_pod = true; gs.rep_pod = p; }                    // core.go:486-488
    if (!gs.pg.has_min_resources) {                                            // core.go:489-493
      gs.pg.has_min_resources = true;
      gs.pg.min_resources.clear();
      for (auto& c : p.containers)
        for (auto& kv : container_demand(c)) gs.pg.min_resources.push_back(kv);
    }
    if (gs.pg.occupied_by.empty() && !p.owner_uids.empty()) gs.pg.occupied_by = joined_sorted(p.owner_uids);  // :496-500
  }
  return Status{};
}

Status BatchSchedulingPlugin::PackNodeRows(const PackedSnapshot& ctx, const std::vector<const NodeInfo*>& rows,
                                           PackedSnapshot* out, bool* needs_full) {
  if (!out || !needs_full) return Status{BS_CODE_ERROR, "PackNodeRows: null output"};
  *needs_full = false;
  PackedSnapshot& ps = *out;
  ps = PackedSnapshot();
  const uint32_t n = (uint32_t)rows.size();
  ps.lanes = ctx.lanes; ps.scalar_names = ctx.scalar_names; ps.sel_pairs = ctx.sel_pairs; ps.taint_list = ctx.taint_list;
  ps.n_nodes = n;
  // affinity verdicts of the changed rows: aff_bits[c * n + k] = 0 / 1 (one word per (class, row); the
  // caller patches the round's bit table with them)
  ps.sel_in_table = ctx.sel_in_table;
  ps.aff_classes = ctx.aff_classes;
  ps.aff_signatures = ctx.aff_signatures;
  ps.aff_bits.assign((size_t)ctx.n_aff() * n, 0);
  for (uint32_t c = 0; c < ctx.n_aff(); ++c)
    for (uint32_t k = 0; k < n; ++k)
      if (rows[k] && rows[k]->node && aff_class_matches(ctx.aff_classes[c], *rows[k]->node)) ps.aff_bits[(size_t)c * n + k] = 1;
  const RowEncoder enc(ctx, ps);
  for (uint32_t i = 0; i < n; ++i) {
    const Encoded r = enc.node(rows[i], i, n);
    if (r == kNeedsFull) { *needs_full = true; return Status{}; }
    if (r != kEncoded) return Status{BS_CODE_ERROR, kEncodeError[r]};
  }
  return Status{};
}

Status BatchSchedulingPlugin::Reevaluate() {
  bs_results r{};
  r.prefilter = prefilter_.data(); r.feasible_count = feasible_.data(); r.best_node = best_node_.data();
  r.admit = admit_.data(); r.new_denied = new_denied_.data(); r.order = order_.data(); r.rank = rank_.data();
  int rc = bs_begin_cycle(eng_, now_ns_);   // matched / flags columns follow the engine's tables at now
  if (!rc) rc = bs_evaluate(eng_, &r);
  if (!rc) rc = FetchTopK();
  if (!rc) rc = FetchReasons();
  if (!rc) rc = FetchPriority();
  if (rc) return Status{BS_CODE_ERROR, std::string("bsched: ") + bs_strerror(rc) + " (" + bs_last_error(eng_) + ")"};
  return Status{};   // (new_denied groups were deny-listed by the engine's fetch, core.go:142,163)
}

int BatchSchedulingPlugin::FetchTopK() {
  if (!topk_) return BS_OK;
  const uint32_t P = packed_.n_pods;
  topk_node_.assign((size_t)P * topk_, -1);
  topk_score_.assign((size_t)P * topk_, INT64_MIN);
  return bs_fetch_topk_rows(eng_, 0, P, topk_node_.data(), topk_score_.data());
}

std::vector<std::pair<std::string, int64_t>> BatchSchedulingPlugin::TopNodes(const std::string& uid) const {
  std::vector<std::pair<std::string, int64_t>> out;
  const int32_t row = pod_row_.find(uid);
  if (row < 0 || !topk_ || topk_node_.size() < ((size_t)row + 1) * topk_) return out;
  for (uint32_t i = 0; i < topk_; ++i) {
    const int32_t n = topk_node_[(size_t)row * topk_ + i];
    if (n < 0) break;   // padding: the pod fits on fewer nodes
    out.emplace_back((size_t)n < node_names_.size() ? node_names_[n] : std::string(), topk_score_[(size_t)row * topk_ + i]);
  }
  return out;
}

int BatchSchedulingPlugin::FetchReasons() {
  if (!(out_flags_ & BS_OUT_REASONS)) return BS_OK;
  const uint32_t P = packed_.n_pods;
  reasons_.assign((size_t)P * (4 + packed_.lanes), 0);
  const int rc = bs_fetch_reason_rows(eng_, 0, P, reasons_.data());
  ipf_reasons_.clear();
  hp_reasons_.clear();
  if (rc) return rc;
  if (interpod_filter_) {
    ipf_reasons_.assign((size_t)P * 3, 0);
    if (int r = bs_fetch_interpod_reason_rows(eng_, 0, P, ipf_reasons_.data())) return r;
  }
  if (!host_port_filter_) return BS_OK;
  hp_reasons_.assign(P, 0);
  return bs_fetch_host_port_reason_rows(eng_, 0, P, hp_reasons_.data());
}

int BatchSchedulingPlugin::FetchPriority() {
  if (!priority_k_) return BS_OK;
  const uint32_t P = packed_.n_pods;
  prio_node_.assign((size_t)P * priority_k_, -1);
  prio_score_.assign((size_t)P * priority_k_, INT64_MIN);
  return bs_fetch_priority_rows(eng_, 0, P, prio_node_.data(), prio_score_.data());
}

std::vector<std::pair<std::string, int64_t>> BatchSchedulingPlugin::PriorityNodes(const std::string& uid) const {
  std::vector<std::pair<std::string, int64_t>> out;
  const int32_t row = pod_row_.find(uid);
  if (row < 0 || !priority_k_ || prio_node_.size() < ((size_t)row + 1) * priority_k_) return out;
  for (uint32_t i = 0; i < priority_k_; ++i) {
    const int32_t n = prio_node_[(size_t)row * priority_k_ + i];
    if (n < 0) break;   // padding: the pod fits on fewer nodes
    out.emplace_back((size_t)n < node_names_.size() ? node_names_[n] : std::string(), prio_score_[(size_t)row * priority_k_ + i]);
  }
  return out;
}

void BatchSchedulingPlugin::SetScoreWeights(uint32_t least, uint32_t most, uint32_t balanced) {
  std::lock_guard<std::mutex> lk(mu_);
  weights_[0] = least; weights_[1] = most; weights_[2] = balanced;
  if (eng_) bs_set_score_weights(eng_, least, most, balanced);
}

Status BatchSchedulingPlugin::SetRatioPriority(uint32_t weight, const std::vector<std::pair<uint32_t, uint32_t>>& shape,
                                               const std::map<std::string, uint32_t>& resources) {
  std::lock_guard<std::mutex> lk(mu_);
  auto bad = [](const std::string& why) { return Status{BS_CODE_ERROR, "SetRatioPriority: " + why}; };
  if (shape.empty() || shape.size() > 101) return bad("the shape needs 1 to 101 points");
  std::vector<uint32_t> util, score;
  for (size_t i = 0; i < shape.size(); ++i) {
    if (shape[i].first > 100 || shape[i].second > 10) return bad("utilization lies in 0..100 and score in 0..10");
    if (i && shape[i].first <= shape[i - 1].first) return bad("utilization must be strictly ascending");
    util.push_back(shape[i].first);
    score.push_back(shape[i].second * 10);   // MaxNodeScore / MaxCustomPriorityScore
  }
  for (auto& kv : resources)
    if (kv.second < 1 || kv.second > 100) return bad("resource weights lie in 1..100 (" + kv.first + ")");
  const uint32_t old_weight = ratio_weight_;
  std::vector<uint32_t> old_util = ratio_util_, old_score = ratio_score_;
  std::map<std::string, uint32_t> old_res = ratio_resources_;
  ratio_weight_ = weight;
  ratio_util_ = util;
  ratio_score_ = score;
  ratio_resources_ = resources.empty() ? std::map<std::string, uint32_t>{{"cpu", 1}, {"memory", 1}} : resources;
  const int rc = eng_ ? PushRatio() : BS_OK;
  if (rc) {
    ratio_weight_ = old_weight; ratio_util_ = old_util; ratio_score_ = old_score; ratio_resources_ = old_res;
    return Status{BS_CODE_ERROR, std::string("bsched: ") + bs_strerror(rc) + " (" + bs_last_error(eng_) + ")"};
  }
  return Status{};
}

int BatchSchedulingPlugin::PushRatio() {
  const uint32_t L = eng_lanes_;
  std::vector<uint32_t> lane_w(L, 0);
  uint32_t absent = 0;
  for (auto& kv : ratio_resources_) {
    int lane = -1;
    if (kv.first == "cpu") lane = 0;
    else if (kv.first == "memory") lane = 1;
    else if (kv.first == "ephemeral-storage") lane = 2;
    else
      for (size_t k = 0; k < packed_.scalar_names.size(); ++k)
        if (packed_.scalar_names[k] == kv.first && 4 + k < L) lane = (int)(4 + k);
    if (lane < 0) absent += kv.second;   // `pods` and names without a lane: capacity 0 on every node
    else lane_w[lane] += kv.second;
  }
  return bs_set_ratio_priority(eng_, ratio_weight_, (uint32_t)ratio_util_.size(), ratio_util_.data(), ratio_score_.data(),
                               L, lane_w.data(), absent);
}

namespace {
// GetNonzeroRequestForResource [upstream, from memory]: the Requests' cpu (MilliValue) / memory (Value), 100 m /
// 200 MiB when the key is absent; a key listed twice counts its last entry, as a map assignment would
constexpr int64_t kDefaultMilliCpuRequest = 100, kDefaultMemoryRequest = 200ll * 1024 * 1024;
bool nonzero_of(const Pod& p, int64_t* cpu, int64_t* mem) {
  *cpu = *mem = 0;
  for (const Container& c : p.containers) {
    const std::string *qc = nullptr, *qm = nullptr;
    for (auto& kv : c.requests) {
      if (kv.first == "cpu") qc = &kv.second;
      else if (kv.first == "memory") qm = &kv.second;
    }
    int64_t vc = kDefaultMilliCpuRequest, vm = kDefaultMemoryRequest;
    if (qc && !QuantityMilliValue(*qc, &vc)) return false;
    if (qm && !QuantityValue(*qm, &vm)) return false;
    *cpu += vc;
    *mem += vm;
  }
  return true;
}
}  // namespace

Status BatchSchedulingPlugin::PackNonZero(const std::vector<const NodeInfo*>& snapshot, const std::vector<const Pod*>& pending,
                                          std::vector<int64_t>* node_nz, std::vector<int64_t>* pod_nz) {
  auto bad = [](const Pod& p) { return Status{BS_CODE_ERROR, "PackNonZero: malformed request quantity in pod " + p.ns + "/" + p.name}; };
  if (node_nz) {
    const size_t N = snapshot.size();
    node_nz->assign(2 * N, 0);
    for (size_t i = 0; i < N; ++i) {
      if (!snapshot[i]) continue;
      for (const Pod* p : snapshot[i]->pods) {   // NodeInfo.NonZeroRequest(): the same sum over the node's pods
        int64_t c, m;
        if (!p) continue;
        if (!nonzero_of(*p, &c, &m)) return bad(*p);
        (*node_nz)[i] += c;
        (*node_nz)[N + i] += m;
      }
    }
  }
  if (pod_nz) {
    const size_t P = pending.size();
    pod_nz->assign(2 * P, 0);
    for (size_t i = 0; i < P; ++i) {
      if (!pending[i]) continue;
      if (!nonzero_of(*pending[i], &(*pod_nz)[i], &(*pod_nz)[P + i])) return bad(*pending[i]);
    }
  }
  return Status{};
}

Status BatchSchedulingPlugin::UploadNonZero(const std::vector<const Pod*>* pending) {
  if (!priority_k_) return Status{};
  std::vector<int64_t> node_nz, pod_nz;
  Status st = PackNonZero(snapshot_, pending ? *pending : std::vector<const Pod*>(), &node_nz, pending ? &pod_nz : nullptr);
  if (!st.ok()) return st;
  int rc = bs_upload_node_nonzero(eng_, (uint32_t)snapshot_.size(), node_nz.data());
  if (!rc && pending) rc = bs_upload_pod_nonzero(eng_, (uint32_t)pending->size(), pod_nz.data());
  if (!rc) rc = bs_set_score_weights(eng_, weights_[0], weights_[1], weights_[2]);
  if (!rc) rc = PushRatio();   // the lanes of this round's scalar resources
  if (rc) return Status{BS_CODE_ERROR, std::string("bsched: ") + bs_strerror(rc) + " (" + bs_last_error(eng_) + ")"};
  return Status{};
}

void BatchSchedulingPlugin::SetNodePriorityWeights(uint32_t taint_toleration, uint32_t node_affinity) {
  std::lock_guard<std::mutex> lk(mu_);
  node_prio_weights_[0] = taint_toleration;
  node_prio_weights_[1] = node_affinity;
}

namespace {
// canonical text of a pod's preferred terms of non-zero weight ("" = none): the class key of PackPreferences
std::string preference_signature(const Pod& p) {
  std::string s;
  for (auto& t : p.preferred_affinity) {
    if (t.weight == 0) continue;   // CalculateNodeAffinityPriorityMap skips it
    s += 'W'; s += std::to_string(t.weight); s += '\x1f';
    for (auto& r : t.preference.match_expressions) {
      s += 'E'; s += r.key; s += '\x1f'; s += r.op; s += '\x1f';
      for (auto& v : r.values) { s += v; s += '\x1d'; }
      s += '\x1e';
    }
  }
  return s;
}
}  // namespace

Status BatchSchedulingPlugin::PackPreferences(const std::vector<const NodeInfo*>& snapshot,
                                              const std::vector<const Pod*>& pending, PackedPreferences* out) {
  if (!out) return Status{BS_CODE_ERROR, "PackPreferences: null output"};
  PackedPreferences& pp = *out;
  pp = PackedPreferences();
  const size_t N = snapshot.size(), P = pending.size();
  // the round's PreferNoSchedule dictionary: one bit per distinct (key, value)
  pp.prefer_taints.assign(N, 0);
  for (size_t i = 0; i < N; ++i) {
    if (!snapshot[i] || !snapshot[i]->node) continue;
    for (const Taint& t : snapshot[i]->node->taints) {
      if (t.effect != "PreferNoSchedule") continue;
      size_t b = 0;
      while (b < pp.taints.size() && !(pp.taints[b].key == t.key && pp.taints[b].value == t.value)) ++b;
      if (b == pp.taints.size()) {
        if (b == 64) return Status{BS_CODE_ERROR, "PackPreferences: more than 64 distinct PreferNoSchedule taints in one round"};
        pp.taints.push_back(t);
      }
      pp.prefer_taints[i] |= 1ull << b;
    }
  }
  // each pod's tolerated bits (getAllTolerationPreferNoSchedule, then ToleratesTaint) and preferred class
  pp.prefer_tol.assign(P, 0);
  pp.pref_class.assign(P, BS_PREF_NONE);
  std::unordered_map<std::string, uint32_t> class_of;
  std::vector<const Pod*> class_pod;   // the first pod of each class
  for (size_t p = 0; p < P; ++p) {
    if (!pending[p]) continue;
    const Pod& pod = *pending[p];
    for (size_t b = 0; b < pp.taints.size(); ++b)
      for (const Toleration& tol : pod.tolerations)
        if ((tol.effect.empty() || tol.effect == "PreferNoSchedule") && tolerates(tol, pp.taints[b])) {
          pp.prefer_tol[p] |= 1ull << b;
          break;
        }
    for (auto& t : pod.preferred_affinity)
      if (t.weight < 0) return Status{BS_CODE_ERROR, "PackPreferences: negative preferred-term weight in pod " + pod.ns + "/" + pod.name};
    std::string sig = preference_signature(pod);
    if (sig.empty()) continue;
    auto it = class_of.find(sig);
    if (it == class_of.end()) {
      it = class_of.emplace(sig, (uint32_t)pp.class_signatures.size()).first;
      pp.class_signatures.push_back(std::move(sig));
      class_pod.push_back(&pod);
    }
    pp.pref_class[p] = it->second;
  }
  // the class x node table: terms whose (non-empty) match_expressions all match the node's labels
  const uint32_t C = pp.n_classes();
  pp.pref_weights.assign((size_t)C * N, 0);
  for (uint32_t c = 0; c < C; ++c)
    for (size_t i = 0; i < N; ++i) {
      if (!snapshot[i] || !snapshot[i]->node) continue;
      const auto& labels = snapshot[i]->node->labels;
      int64_t sum = 0;
      for (auto& t : class_pod[c]->preferred_affinity) {
        if (t.weight == 0 || t.preference.match_expressions.empty()) continue;   // labels.Nothing()
        bool ok = true, valid = true;
        for (auto& r : t.preference.match_expressions) {
          ok = requirement_matches(r, labels, &valid) && valid;   // an invalid requirement: the term counts 0
          if (!ok) break;
        }
        if (ok) sum += t.weight;
      }
      if (sum > INT32_MAX) return Status{BS_CODE_ERROR, "PackPreferences: preferred-term weights above INT32_MAX"};
      pp.pref_weights[(size_t)c * N + i] = (int32_t)sum;
    }
  return Status{};
}

Status BatchSchedulingPlugin::UploadPreferences() {
  if (!priority_k_) return Status{};
  auto fail = [&](int rc) {
    return Status{BS_CODE_ERROR, std::string("bsched: ") + bs_strerror(rc) + " (" + bs_last_error(eng_) + ")"};
  };
  int rc = bs_set_node_priority_weights(eng_, node_prio_weights_[0], node_prio_weights_[1]);
  if (rc) return fail(rc);
  if (!node_prio_weights_[0] && !node_prio_weights_[1]) return Status{};
  PackedPreferences pp;
  Status st = PackPreferences(snapshot_, pending_, &pp);
  if (!st.ok()) return st;
  rc = bs_upload_node_preferences(eng_, (uint32_t)snapshot_.size(), pp.prefer_taints.data(), pp.n_classes(),
                                  pp.pref_weights.data());
  if (!rc) rc = bs_upload_pod_preferences(eng_, (uint32_t)pending_.size(), pp.prefer_tol.data(), pp.pref_class.data());
  return rc ? fail(rc) : Status{};
}

void BatchSchedulingPlugin::SetLocalityWeights(uint32_t image_locality, uint32_t prefer_avoid_pods) {
  std::lock_guard<std::mutex> lk(mu_);
  locality_weights_[0] = image_locality;
  locality_weights_[1] = prefer_avoid_pods;
}

std::string normalized_image_name(const std::string& name) {
  const size_t colon = name.rfind(':'), slash = name.rfind('/');
  // strings.LastIndex gives -1 where rfind gives npos: compare as "position + 1"
  const size_t c1 = colon == std::string::npos ? 0 : colon + 1, s1 = slash == std::string::npos ? 0 : slash + 1;
  return c1 <= s1 ? name + ":latest" : name;
}

namespace {
bool rc_or_rs(const std::string& kind) { return kind == "ReplicationController" || kind == "ReplicaSet"; }
}  // namespace

Status BatchSchedulingPlugin::PackLocality(const std::vector<const NodeInfo*>& snapshot,
                                           const std::vector<const Pod*>& pending, PackedLocality* out) {
  if (!out) return Status{BS_CODE_ERROR, "PackLocality: null output"};
  PackedLocality& pl = *out;
  pl = PackedLocality();
  const size_t N = snapshot.size(), P = pending.size(), W = (N + 31) / 32;
  // the names some pending pod's normalized container image asks for
  std::unordered_map<std::string, uint32_t> wanted;   // name -> dictionary id (UINT32_MAX: not reported yet)
  for (const Pod* pod : pending)
    if (pod)
      for (const Container& c : pod->containers) wanted.emplace(normalized_image_name(c.image), UINT32_MAX);
  // the dictionary in node order: a name's size is the first (lowest-index) node's that reports it
  for (size_t i = 0; i < N; ++i) {
    if (!snapshot[i] || !snapshot[i]->node) continue;
    for (const ContainerImage& im : snapshot[i]->node->images)
      for (const std::string& name : im.names) {
        auto it = wanted.find(name);
        if (it == wanted.end()) continue;
        if (it->second == UINT32_MAX) {
          if (im.size_bytes < 0 || im.size_bytes > BS_IMAGE_SIZE_MAX)
            return Status{BS_CODE_ERROR, "PackLocality: image " + name + " has a size outside [0, 2^48]"};
          it->second = (uint32_t)pl.names.size();
          pl.names.push_back(name);
          pl.image_size.push_back(im.size_bytes);
          pl.image_bits.resize(pl.image_bits.size() + W, 0u);
        }
        pl.image_bits[(size_t)it->second * W + i / 32] |= 1u << (i % 32);
      }
  }
  // each pod's class: its containers' dictionary ids, sorted (a repeated image stays repeated), deduplicated
  pl.image_class.assign(P, BS_IMAGE_NONE);
  std::map<std::vector<uint32_t>, uint32_t> class_of;
  for (size_t p = 0; p < P; ++p) {
    if (!pending[p]) continue;
    std::vector<uint32_t> ids;
    for (const Container& c : pending[p]->containers) {
      const uint32_t id = wanted.at(normalized_image_name(c.image));
      if (id != UINT32_MAX) ids.push_back(id);
    }
    if (ids.empty()) continue;
    if (ids.size() > BS_LOC_CLASS_MAX)
      return Status{BS_CODE_ERROR, "PackLocality: pod " + pending[p]->ns + "/" + pending[p]->name +
                                       " has more than 64 containers with reported images"};
    std::sort(ids.begin(), ids.end());
    auto it = class_of.find(ids);
    if (it == class_of.end()) {
      it = class_of.emplace(ids, pl.n_classes()).first;
      pl.class_images.insert(pl.class_images.end(), ids.begin(), ids.end());
      pl.class_offset.push_back((uint32_t)pl.class_images.size());
    }
    pl.image_class[p] = it->second;
  }
  // the avoid dictionary: RC / RS controllers of pending pods that some node's annotation lists, in node order
  std::set<std::pair<std::string, std::string>> controlling;
  for (const Pod* pod : pending)
    if (pod && rc_or_rs(pod->controller_kind)) controlling.emplace(pod->controller_kind, pod->controller_uid);
  pl.avoid_mask.assign(N, 0);
  std::map<std::pair<std::string, std::string>, uint32_t> bit_of;
  for (size_t i = 0; i < N; ++i) {
    if (!snapshot[i] || !snapshot[i]->node) continue;
    for (const PodController& pc : snapshot[i]->node->prefer_avoid_pods) {
      const auto key = std::make_pair(pc.kind, pc.uid);
      if (!controlling.count(key)) continue;
      auto it = bit_of.find(key);
      if (it == bit_of.end()) {
        if (pl.controllers.size() == 64)
          return Status{BS_CODE_ERROR, "PackLocality: more than 64 avoided controllers of pending pods in one round"};
        it = bit_of.emplace(key, (uint32_t)pl.controllers.size()).first;
        pl.controllers.push_back(pc);
      }
      pl.avoid_mask[i] |= 1ull << it->second;
    }
  }
  pl.avoid_bit.assign(P, BS_AVOID_NONE);
  for (size_t p = 0; p < P; ++p) {
    if (!pending[p] || !rc_or_rs(pending[p]->controller_kind)) continue;
    auto it = bit_of.find(std::make_pair(pending[p]->controller_kind, pending[p]->controller_uid));
    if (it != bit_of.end()) pl.avoid_bit[p] = (uint8_t)it->second;
  }
  return Status{};
}

Status BatchSchedulingPlugin::UploadLocality() {
  if (!priority_k_) return Status{};
  auto fail = [&](int rc) {
    return Status{BS_CODE_ERROR, std::string("bsched: ") + bs_strerror(rc) + " (" + bs_last_error(eng_) + ")"};
  };
  int rc = bs_set_locality_weights(eng_, locality_weights_[0], locality_weights_[1]);
  if (rc) return fail(rc);
  if (!locality_weights_[0] && !locality_weights_[1]) return Status{};
  PackedLocality pl;
  Status st = PackLocality(snapshot_, pending_, &pl);
  if (!st.ok()) return st;
  // empty vectors may have null data(): the parts are present, so point them at something
  static const uint64_t none = 0;
  auto nz = [](const void* p) { return p ? p : (const void*)&none; };
  rc = bs_upload_node_locality(eng_, (uint32_t)snapshot_.size(), (uint32_t)pl.names.size(),
                               (const int64_t*)nz(pl.image_size.data()), (const uint32_t*)nz(pl.image_bits.data()),
                               (const uint64_t*)nz(pl.avoid_mask.data()));
  if (!rc)
    rc = bs_upload_pod_locality(eng_, (uint32_t)pending_.size(), (const uint32_t*)nz(pl.image_class.data()),
                                pl.n_classes(), pl.class_offset.data(), (const uint32_t*)nz(pl.class_images.data()),
                                (const uint8_t*)nz(pl.avoid_bit.data()));
  return rc ? fail(rc) : Status{};
}

void BatchSchedulingPlugin::SetSpreadSelectors(SpreadSelectors selectors) {
  std::lock_guard<std::mutex> lk(mu_);
  spread_selectors_ = std::move(selectors);
}

void BatchSchedulingPlugin::SetPodDisruptionBudgets(std::vector<PodDisruptionBudget> pdbs) {
  std::lock_guard<std::mutex> lk(mu_);
  pdbs_ = std::move(pdbs);
}

void BatchSchedulingPlugin::SetSelectorSpreadWeight(uint32_t selector_spread) {
  std::lock_guard<std::mutex> lk(mu_);
  spread_weight_ = selector_spread;
}

namespace {
// one requirement of a converted selector (labels.Requirement): Equals from a map or matchLabels, or a
// LabelSelectorRequirement's operator
struct SpreadReq {
  std::string key, op;
  std::vector<std::string> values;   // sorted: the set of the requirement
};
using SpreadSel = std::vector<SpreadReq>;   // ANDed; sorted by key, then operator

bool spread_req_matches(const SpreadReq& r, const std::map<std::string, std::string>& labels) {
  const auto it = labels.find(r.key);
  const bool has = it != labels.end();
  auto in = [&] { return has && std::binary_search(r.values.begin(), r.values.end(), it->second); };
  if (r.op == "=" || r.op == "In") return in();
  if (r.op == "NotIn") return !in();
  if (r.op == "Exists") return has;
  return !has;   // DoesNotExist
}
bool spread_sel_matches(const SpreadSel& s, const std::map<std::string, std::string>& labels) {
  for (const SpreadReq& r : s)
    if (!spread_req_matches(r, labels)) return false;
  return true;
}
void sort_sel(SpreadSel* s) {
  for (SpreadReq& r : *s) std::sort(r.values.begin(), r.values.end());
  std::sort(s->begin(), s->end(), [](const SpreadReq& a, const SpreadReq& b) {
    return a.key != b.key ? a.key < b.key : a.op != b.op ? a.op < b.op : a.values < b.values;
  });
}
// labels.SelectorFromSet of a Service or RC selector (an empty map: Everything)
SpreadSel sel_from_map(const std::map<std::string, std::string>& m) {
  SpreadSel s;
  for (auto& kv : m) s.push_back(SpreadReq{kv.first, "=", {kv.second}});
  return s;
}
// metav1.LabelSelectorAsSelector of a non-nil selector; false when a requirement fails to convert
bool sel_from_label_selector(const LabelSelector& ls, SpreadSel* out) {
  SpreadSel s = sel_from_map(ls.match_labels);
  for (const LabelSelectorRequirement& r : ls.match_expressions) {
    if (r.op == "In" || r.op == "NotIn") {
      if (r.values.empty()) return false;
    } else if (r.op == "Exists" || r.op == "DoesNotExist") {
      if (!r.values.empty()) return false;
    } else {
      return false;
    }
    s.push_back(SpreadReq{r.key, r.op, r.values});
  }
  sort_sel(&s);
  *out = std::move(s);
  return true;
}
// the canonical text of a converted selector (a class key part)
std::string sel_text(const SpreadSel& s) {
  std::string t;
  for (const SpreadReq& r : s) {
    t += r.key; t += '\x1f'; t += r.op; t += '\x1f';
    for (auto& v : r.values) { t += v; t += '\x1d'; }
    t += '\x1e';
  }
  return t;
}
}  // namespace

Status BatchSchedulingPlugin::PackSpread(const std::vector<const NodeInfo*>& snapshot,
                                         const std::vector<const Pod*>& pending, const SpreadSelectors& selectors,
                                         PackedSpread* out) {
  if (!out) return Status{BS_CODE_ERROR, "PackSpread: null output"};
  PackedSpread& ps = *out;
  ps = PackedSpread();
  const size_t N = snapshot.size(), P = pending.size();
  // the zone dictionary (utilnode.GetZoneKey: the beta region and zone labels), in order of first appearance
  ps.zone.assign(N, BS_ZONE_NONE);
  std::unordered_map<std::string, uint8_t> zone_of;
  for (size_t i = 0; i < N; ++i) {
    if (!snapshot[i] || !snapshot[i]->node) continue;
    const auto& labels = snapshot[i]->node->labels;
    const auto r = labels.find("failure-domain.beta.kubernetes.io/region");
    const auto z = labels.find("failure-domain.beta.kubernetes.io/zone");
    const std::string region = r == labels.end() ? "" : r->second, zone = z == labels.end() ? "" : z->second;
    if (region.empty() && zone.empty()) continue;
    const std::string key = region + std::string(":\0:", 3) + zone;
    auto it = zone_of.find(key);
    if (it == zone_of.end()) {
      if (ps.zones.size() == BS_SPREAD_ZONE_MAX)
        return Status{BS_CODE_ERROR, "PackSpread: more than 64 zones in one round"};
      it = zone_of.emplace(key, (uint8_t)ps.zones.size()).first;
      ps.zones.push_back(key);
    }
    ps.zone[i] = it->second;
  }
  // the converted selectors of the listers' objects, once: (namespace, selector) of those that can select a pod
  struct Cand {
    const std::string* ns;
    SpreadSel sel;
    bool needs_labels;   // RC / RS / StatefulSet: their listers return an error for a pod without labels
  };
  std::vector<Cand> cands;
  for (const Service& s : selectors.services)
    if (s.has_selector) cands.push_back(Cand{&s.ns, sel_from_map(s.selector), false});   // nil: matches nothing
  for (const ReplicationController& c : selectors.controllers)
    if (c.has_selector && !c.selector.empty()) cands.push_back(Cand{&c.ns, sel_from_map(c.selector), true});
  auto add_ls = [&](const std::string& ns, bool has, const LabelSelector& ls) {
    if (!has || (ls.match_labels.empty() && ls.match_expressions.empty())) return;   // nil or empty: nothing
    SpreadSel s;
    if (sel_from_label_selector(ls, &s)) cands.push_back(Cand{&ns, std::move(s), true});
  };
  for (const ReplicaSet& r : selectors.replica_sets) add_ls(r.ns, r.has_selector, r.selector);
  for (const StatefulSet& r : selectors.stateful_sets) add_ls(r.ns, r.has_selector, r.selector);
  // each pod's class: its namespace and the sorted set of its selectors' texts
  ps.spread_class.assign(P, BS_SPREAD_NONE);
  std::unordered_map<std::string, uint32_t> class_of;
  std::vector<std::pair<const std::string*, std::vector<const SpreadSel*>>> class_sels;
  for (size_t p = 0; p < P; ++p) {
    if (!pending[p]) continue;
    const Pod& pod = *pending[p];
    std::vector<std::pair<std::string, const SpreadSel*>> mine;
    for (const Cand& c : cands)
      if (*c.ns == pod.ns && (!c.needs_labels || !pod.labels.empty()) && spread_sel_matches(c.sel, pod.labels))
        mine.emplace_back(sel_text(c.sel), &c.sel);
    if (mine.empty()) continue;
    std::sort(mine.begin(), mine.end(), [](auto& a, auto& b) { return a.first < b.first; });
    mine.erase(std::unique(mine.begin(), mine.end(), [](auto& a, auto& b) { return a.first == b.first; }), mine.end());
    std::string sig = pod.ns;
    for (auto& m : mine) { sig += '\x1c'; sig += m.first; }
    auto it = class_of.find(sig);
    if (it == class_of.end()) {
      it = class_of.emplace(sig, ps.n_classes()).first;
      ps.class_signatures.push_back(std::move(sig));
      std::vector<const SpreadSel*> sels;
      for (auto& m : mine) sels.push_back(m.second);
      class_sels.emplace_back(&pod.ns, std::move(sels));
    }
    ps.spread_class[p] = it->second;
  }
  // countMatchingPods over NodeInfo::pods
  const uint32_t C = ps.n_classes();
  ps.counts.assign((size_t)C * N, 0);
  for (uint32_t c = 0; c < C; ++c)
    for (size_t i = 0; i < N; ++i) {
      if (!snapshot[i]) continue;
      int64_t n = 0;
      for (const Pod* bp : snapshot[i]->pods) {
        if (!bp || bp->ns != *class_sels[c].first || bp->terminating) continue;
        bool ok = true;
        for (const SpreadSel* s : class_sels[c].second)
          if (!spread_sel_matches(*s, bp->labels)) { ok = false; break; }
        n += ok;
      }
      if (n > BS_SPREAD_COUNT_MAX) return Status{BS_CODE_ERROR, "PackSpread: a count above BS_SPREAD_COUNT_MAX"};
      ps.counts[(size_t)c * N + i] = (int32_t)n;
    }
  return Status{};
}

Status BatchSchedulingPlugin::UploadSpread() {
  if (!priority_k_) return Status{};
  auto fail = [&](int rc) {
    return Status{BS_CODE_ERROR, std::string("bsched: ") + bs_strerror(rc) + " (" + bs_last_error(eng_) + ")"};
  };
  int rc = bs_set_spread_weight(eng_, spread_weight_);
  if (rc) return fail(rc);
  if (!spread_weight_) return Status{};
  PackedSpread ps;
  Status st = PackSpread(snapshot_, pending_, spread_selectors_, &ps);
  if (!st.ok()) return st;
  rc = bs_upload_node_spread(eng_, (uint32_t)snapshot_.size(), (uint32_t)ps.zones.size(), ps.zone.data(), ps.n_classes(),
                             ps.counts.data());
  if (!rc) rc = bs_upload_pod_spread(eng_, (uint32_t)pending_.size(), ps.spread_class.data());
  return rc ? fail(rc) : Status{};
}

void BatchSchedulingPlugin::SetInterPodAffinityWeight(uint32_t inter_pod_affinity) {
  std::lock_guard<std::mutex> lk(mu_);
  interpod_weight_ = inter_pod_affinity;
}

Status BatchSchedulingPlugin::SetHardPodAffinityWeight(int32_t hard_pod_affinity_weight) {
  if (hard_pod_affinity_weight < 0 || hard_pod_affinity_weight > 100)
    return Status{BS_CODE_ERROR, "SetHardPodAffinityWeight: the weight is outside 0..100"};
  std::lock_guard<std::mutex> lk(mu_);
  hard_pod_affinity_weight_ = hard_pod_affinity_weight;
  return Status{};
}

namespace {
// A pod-affinity term as the inter-pod dictionaries identify it: its namespaces resolved (empty: the owner's), sorted
// and deduplicated; its selector converted by SelectorSpread's rules (has_sel = false: nil; ok = false: it fails to
// convert); and the signature of the three with the key.
struct ResolvedTerm {
  bool has_sel = false, ok = true;
  SpreadSel sel;
  std::vector<std::string> ns;
  std::string sig;
};
ResolvedTerm resolve_term(const PodAffinityTerm& t, const std::string& owner_ns) {
  ResolvedTerm r;
  r.has_sel = t.has_selector;
  r.ok = !t.has_selector || sel_from_label_selector(t.selector, &r.sel);
  r.ns = t.namespaces.empty() ? std::vector<std::string>{owner_ns} : t.namespaces;
  std::sort(r.ns.begin(), r.ns.end());
  r.ns.erase(std::unique(r.ns.begin(), r.ns.end()), r.ns.end());
  for (auto& n : r.ns) { r.sig += n; r.sig += '\x1d'; }
  r.sig += '\x1c';
  r.sig += !r.ok ? std::string("bad") : t.has_selector ? "sel:" + sel_text(r.sel) : std::string("nil");
  r.sig += '\x1c';
  r.sig += t.topology_key;
  return r;
}
bool pod_matches_term(const Pod& pod, const ResolvedTerm& r) {
  return r.has_sel && r.ok && std::binary_search(r.ns.begin(), r.ns.end(), pod.ns) && spread_sel_matches(r.sel, pod.labels);
}
// each key's values over the nodes with a Node(), in order of first appearance; topo [keys][nodes]
void number_topology(const std::vector<const NodeInfo*>& snapshot, const std::vector<std::string>& keys,
                     std::vector<std::vector<std::string>>* values, std::vector<uint32_t>* n_values,
                     std::vector<uint32_t>* topo) {
  const size_t K = keys.size(), N = snapshot.size();
  values->assign(K, {});
  n_values->assign(K, 0);
  topo->assign(K * N, BS_TOPO_NONE);
  for (size_t k = 0; k < K; ++k) {
    std::unordered_map<std::string, uint32_t> value_of;
    for (size_t i = 0; i < N; ++i) {
      if (!snapshot[i] || !snapshot[i]->node) continue;
      const auto& labels = snapshot[i]->node->labels;
      const auto l = labels.find(keys[k]);
      if (l == labels.end()) continue;
      auto it = value_of.find(l->second);
      if (it == value_of.end()) {
        it = value_of.emplace(l->second, (uint32_t)(*values)[k].size()).first;
        (*values)[k].push_back(l->second);
      }
      (*topo)[k * N + i] = it->second;
    }
    (*n_values)[k] = (uint32_t)(*values)[k].size();
  }
}
}  // namespace

Status BatchSchedulingPlugin::PackInterPodAffinity(const std::vector<const NodeInfo*>& snapshot,
                                                   const std::vector<const Pod*>& pending, int32_t hard_weight,
                                                   PackedInterPodAffinity* out) {
  if (!out) return Status{BS_CODE_ERROR, "PackInterPodAffinity: null output"};
  PackedInterPodAffinity& pk = *out;
  pk = PackedInterPodAffinity();
  const size_t N = snapshot.size(), P = pending.size();
  // the dictionaries: keys and terms in order of first appearance; a term keeps its converted selector (nullopt: nil)
  // and its resolved namespaces for the match tests
  struct TermInfo {
    bool has_sel;
    SpreadSel sel;
    std::vector<std::string> ns;   // sorted
  };
  std::unordered_map<std::string, uint32_t> key_of, term_of;
  std::vector<TermInfo> terms;
  // the (term, signed weight) pairs a pod's processing reads; bad = a term's selector fails to convert
  auto own_of = [&](const Pod& pod, bool bound_side, std::map<uint32_t, int64_t>* own, bool* bad) -> Status {
    auto add = [&](const PodAffinityTerm& t, int64_t w) -> Status {
      ResolvedTerm r = resolve_term(t, pod.ns);
      if (!r.ok) {
        *bad = true;
        return Status{};
      }
      if (t.topology_key.empty()) return Status{};   // NodesHaveSameTopologyKey never holds
      const std::string& sig = r.sig;
      auto kit = key_of.find(t.topology_key);
      if (kit == key_of.end()) {
        if (pk.keys.size() == BS_IPA_KEY_MAX)
          return Status{BS_CODE_ERROR, "PackInterPodAffinity: more than BS_IPA_KEY_MAX topology keys"};
        kit = key_of.emplace(t.topology_key, (uint32_t)pk.keys.size()).first;
        pk.keys.push_back(t.topology_key);
      }
      auto it = term_of.find(sig);
      if (it == term_of.end()) {
        it = term_of.emplace(sig, (uint32_t)terms.size()).first;
        terms.push_back(TermInfo{t.has_selector, std::move(r.sel), std::move(r.ns)});
        pk.term_signatures.push_back(sig);
        pk.term_key.push_back(kit->second);
      }
      (*own)[it->second] += w;
      return Status{};
    };
    Status st;
    if (bound_side && hard_weight > 0)
      for (const PodAffinityTerm& t : pod.required_pod_affinity)
        if (!(st = add(t, hard_weight)).ok()) return st;
    for (const WeightedPodAffinityTerm& t : pod.preferred_pod_affinity)
      if (!(st = add(t.term, t.weight)).ok()) return st;
    for (const WeightedPodAffinityTerm& t : pod.preferred_pod_anti_affinity)
      if (!(st = add(t.term, -(int64_t)t.weight)).ok()) return st;
    return Status{};
  };
  std::vector<const Pod*> bound;
  std::vector<std::map<uint32_t, int64_t>> bown, pown(P);
  bool invalid_bound = false;
  Status st;
  for (size_t i = 0; i < N; ++i) {
    if (!snapshot[i] || !snapshot[i]->node) continue;
    for (const Pod* bp : snapshot[i]->pods) {
      if (!bp) continue;
      if (bound.size() == BS_IPA_BOUND_MAX)
        return Status{BS_CODE_ERROR, "PackInterPodAffinity: more than BS_IPA_BOUND_MAX bound pods"};
      bound.push_back(bp);
      pk.bound_node.push_back((uint32_t)i);
      bown.emplace_back();
      bool bad = false;
      if (!(st = own_of(*bp, true, &bown.back(), &bad)).ok()) return st;
      invalid_bound = invalid_bound || bad;
    }
  }
  std::vector<uint8_t> pbad(P, 0);
  for (size_t p = 0; p < P; ++p) {
    if (!pending[p]) continue;
    bool bad = false;
    if (!(st = own_of(*pending[p], false, &pown[p], &bad)).ok()) return st;
    pbad[p] = bad && !bound.empty();
  }
  // the terms each side owns: a pod's match entries are the other side's terms it matches
  std::vector<uint32_t> b_terms, p_terms;
  {
    std::vector<uint8_t> in_b(terms.size(), 0), in_p(terms.size(), 0);
    for (auto& o : bown) for (auto& kv : o) in_b[kv.first] = 1;
    for (auto& o : pown) for (auto& kv : o) in_p[kv.first] = 1;
    for (uint32_t t = 0; t < terms.size(); ++t) {
      if (in_b[t]) b_terms.push_back(t);
      if (in_p[t]) p_terms.push_back(t);
    }
  }
  auto matches = [&](const Pod& pod, uint32_t t) {
    const TermInfo& ti = terms[t];
    return ti.has_sel && std::binary_search(ti.ns.begin(), ti.ns.end(), pod.ns) && spread_sel_matches(ti.sel, pod.labels);
  };
  // a pod's sorted entries as a class, in order of first appearance; no entries: BS_IPA_NONE
  auto classify = [&](const Pod& pod, const std::map<uint32_t, int64_t>& own, const std::vector<uint32_t>& other,
                      std::map<std::vector<std::tuple<uint32_t, int32_t, uint8_t>>, uint32_t>& class_of,
                      PackedInterPodAffinity::Classes& cl, uint32_t* out_class) -> Status {
    std::map<uint32_t, std::pair<int64_t, uint8_t>> ent;
    for (auto& kv : own) ent[kv.first].first = kv.second;
    for (uint32_t t : other)
      if (matches(pod, t)) ent[t].second = 1;
    std::vector<std::tuple<uint32_t, int32_t, uint8_t>> key;
    for (auto& kv : ent) {
      if (!kv.second.first && !kv.second.second) continue;
      if (kv.second.first < -BS_IPA_OWN_MAX || kv.second.first > BS_IPA_OWN_MAX)
        return Status{BS_CODE_ERROR, "PackInterPodAffinity: a pod's summed weight on one term exceeds BS_IPA_OWN_MAX"};
      key.emplace_back(kv.first, (int32_t)kv.second.first, kv.second.second);
    }
    if (key.size() > BS_IPA_CLASS_MAX)
      return Status{BS_CODE_ERROR, "PackInterPodAffinity: a pod lists more than BS_IPA_CLASS_MAX terms"};
    *out_class = BS_IPA_NONE;
    if (key.empty()) return Status{};
    auto it = class_of.find(key);
    if (it == class_of.end()) {
      it = class_of.emplace(key, cl.n_classes()).first;
      for (auto& e : key) {
        cl.term.push_back(std::get<0>(e));
        cl.own.push_back(std::get<1>(e));
        cl.match.push_back(std::get<2>(e));
      }
      cl.offset.push_back((uint32_t)cl.term.size());
    }
    *out_class = it->second;
    return Status{};
  };
  std::map<std::vector<std::tuple<uint32_t, int32_t, uint8_t>>, uint32_t> bclass_of, pclass_of;
  pk.bound_class.assign(bound.size(), BS_IPA_NONE);
  for (size_t k = 0; k < bound.size(); ++k)
    if (!(st = classify(*bound[k], bown[k], p_terms, bclass_of, pk.bound_classes, &pk.bound_class[k])).ok()) return st;
  pk.pod_class.assign(P, BS_IPA_NONE);
  for (size_t p = 0; p < P; ++p)
    if (pending[p] && !invalid_bound && !pbad[p])
      if (!(st = classify(*pending[p], pown[p], b_terms, pclass_of, pk.pod_classes, &pk.pod_class[p])).ok()) return st;
  number_topology(snapshot, pk.keys, &pk.values, &pk.n_values, &pk.topo);
  return Status{};
}

void BatchSchedulingPlugin::SetInterPodAffinityFilter(bool on) {
  std::lock_guard<std::mutex> lk(mu_);
  interpod_filter_ = on;
}

void BatchSchedulingPlugin::SetInterPodAffinityFilterInWalks(bool on) {
  std::lock_guard<std::mutex> lk(mu_);
  interpod_filter_walks_ = on;
}

Status BatchSchedulingPlugin::PackInterPodFilter(const std::vector<const NodeInfo*>& snapshot,
                                                 const std::vector<const Pod*>& pending, PackedInterPodFilter* out,
                                                 bool placed) {
  if (!out) return Status{BS_CODE_ERROR, "PackInterPodFilter: null output"};
  PackedInterPodFilter& pk = *out;
  pk = PackedInterPodFilter();
  const size_t N = snapshot.size(), P = pending.size();
  std::unordered_map<std::string, uint32_t> key_of, term_of;
  // the dictionary term of signature `sig` (role-prefixed) on `key`; fresh: it is new
  auto term_id = [&](const std::string& sig, const std::string& key, uint32_t* id, bool* fresh) -> Status {
    auto kit = key_of.find(key);
    if (kit == key_of.end()) {
      if (pk.keys.size() == BS_IPA_KEY_MAX)
        return Status{BS_CODE_ERROR, "PackInterPodFilter: more than BS_IPA_KEY_MAX topology keys"};
      kit = key_of.emplace(key, (uint32_t)pk.keys.size()).first;
      pk.keys.push_back(key);
    }
    auto it = term_of.find(sig);
    *fresh = it == term_of.end();
    if (*fresh) {
      it = term_of.emplace(sig, (uint32_t)pk.term_key.size()).first;
      pk.term_signatures.push_back(sig);
      pk.term_key.push_back(kit->second);
    }
    *id = it->second;
    return Status{};
  };
  // bound pods and their required anti-affinity terms (own = 1)
  std::vector<const Pod*> bound;
  std::vector<std::map<uint32_t, std::pair<int32_t, uint8_t>>> bent;   // term -> (own, match)
  std::vector<std::pair<ResolvedTerm, uint32_t>> existing;             // distinct existing anti terms and their ids
  Status st;
  for (size_t i = 0; i < N; ++i) {
    if (!snapshot[i] || !snapshot[i]->node) continue;
    for (const Pod* bp : snapshot[i]->pods) {
      if (!bp) continue;
      if (bound.size() == BS_IPF_BOUND_MAX)
        return Status{BS_CODE_ERROR, "PackInterPodFilter: more than BS_IPF_BOUND_MAX bound pods"};
      bound.push_back(bp);
      pk.bound_node.push_back((uint32_t)i);
      bent.emplace_back();
      for (const PodAffinityTerm& t : bp->required_pod_anti_affinity) {
        ResolvedTerm r = resolve_term(t, bp->ns);
        uint32_t id;
        bool fresh;
        if (!(st = term_id("x\x1e" + r.sig, t.topology_key, &id, &fresh)).ok()) return st;
        if (fresh) existing.emplace_back(std::move(r), id);
        bent.back()[id].first = 1;
      }
    }
  }
  // pending pods: EXISTING entries, the affinity set's terms, the anti-affinity terms
  struct Set { std::vector<ResolvedTerm> terms; std::vector<uint32_t> ids; };
  std::vector<Set> sets;
  std::vector<std::pair<ResolvedTerm, uint32_t>> antis;
  std::unordered_map<std::string, size_t> set_of;
  std::map<std::pair<std::vector<std::pair<uint32_t, uint8_t>>, uint8_t>, uint32_t> class_of;
  std::vector<std::vector<uint32_t>> own_anti(placed ? P : 0);   // placed: each pending pod's anti-affinity terms
  pk.pod_class.assign(P, BS_IPF_NONE);
  for (size_t p = 0; p < P; ++p) {
    if (!pending[p]) continue;
    const Pod& pod = *pending[p];
    std::set<std::pair<uint32_t, uint8_t>> ent;
    for (auto& e : existing)
      if (pod_matches_term(pod, e.first)) ent.emplace(e.second, (uint8_t)BS_IPF_EXISTING);
    uint8_t self = 0;
    if (!pod.required_pod_affinity.empty()) {
      Set set;
      std::string ssig;
      for (const PodAffinityTerm& t : pod.required_pod_affinity) {
        set.terms.push_back(resolve_term(t, pod.ns));
        ssig += set.terms.back().sig;
        ssig += '\x1f';
      }
      auto it = set_of.find(ssig);
      if (it == set_of.end()) {
        for (size_t k = 0; k < set.terms.size(); ++k) {
          uint32_t id;
          bool fresh;
          if (!(st = term_id("a\x1e" + ssig + "\x1e" + std::to_string(k), pod.required_pod_affinity[k].topology_key,
                             &id, &fresh)).ok())
            return st;
          set.ids.push_back(id);
        }
        it = set_of.emplace(ssig, sets.size()).first;
        sets.push_back(std::move(set));
      }
      const Set& s = sets[it->second];
      self = 1;
      for (size_t k = 0; k < s.terms.size(); ++k) {
        ent.emplace(s.ids[k], (uint8_t)BS_IPF_AFFINITY);
        self = self && pod_matches_term(pod, s.terms[k]);
      }
    }
    for (const PodAffinityTerm& t : pod.required_pod_anti_affinity) {
      ResolvedTerm r = resolve_term(t, pod.ns);
      uint32_t id;
      bool fresh;
      if (!(st = term_id("n\x1e" + r.sig, t.topology_key, &id, &fresh)).ok()) return st;
      if (fresh) antis.emplace_back(std::move(r), id);
      ent.emplace(id, (uint8_t)BS_IPF_ANTI);
      if (placed) own_anti[p].push_back(id);
    }
    if (ent.empty()) continue;
    if (ent.size() > BS_IPF_CLASS_MAX)
      return Status{BS_CODE_ERROR, "PackInterPodFilter: a pod lists more than BS_IPF_CLASS_MAX terms"};
    auto key = std::make_pair(std::vector<std::pair<uint32_t, uint8_t>>(ent.begin(), ent.end()), self);
    auto it = class_of.find(key);
    if (it == class_of.end()) {
      it = class_of.emplace(key, pk.n_pod_classes()).first;
      for (auto& e : key.first) {
        pk.pod_term.push_back(e.first);
        pk.pod_role.push_back(e.second);
      }
      pk.pod_offset.push_back((uint32_t)pk.pod_term.size());
      pk.self_match.push_back(self);
    }
    pk.pod_class[p] = it->second;
  }
  // the bound pods' match entries: a set's terms when they match the whole set, an anti term when they match it
  for (size_t k = 0; k < bound.size(); ++k) {
    for (const Set& s : sets) {
      bool all = true;
      for (const ResolvedTerm& r : s.terms) all = all && pod_matches_term(*bound[k], r);
      if (all)
        for (uint32_t id : s.ids) bent[k][id].second = 1;
    }
    for (auto& a : antis)
      if (pod_matches_term(*bound[k], a.first)) bent[k][a.second].second = 1;
  }
  std::map<std::vector<std::tuple<uint32_t, int32_t, uint8_t>>, uint32_t> bclass_of;
  pk.bound_class.assign(bound.size(), BS_IPF_NONE);
  for (size_t k = 0; k < bound.size(); ++k) {
    if (bent[k].empty()) continue;
    if (bent[k].size() > BS_IPF_CLASS_MAX)
      return Status{BS_CODE_ERROR, "PackInterPodFilter: a bound pod lists more than BS_IPF_CLASS_MAX terms"};
    std::vector<std::tuple<uint32_t, int32_t, uint8_t>> key;
    for (auto& kv : bent[k]) key.emplace_back(kv.first, kv.second.first, kv.second.second);
    auto it = bclass_of.find(key);
    if (it == bclass_of.end()) {
      PackedInterPodAffinity::Classes& cl = pk.bound_classes;
      it = bclass_of.emplace(key, cl.n_classes()).first;
      for (auto& e : key) {
        cl.term.push_back(std::get<0>(e));
        cl.own.push_back(std::get<1>(e));
        cl.match.push_back(std::get<2>(e));
      }
      cl.offset.push_back((uint32_t)cl.term.size());
    }
    pk.bound_class[k] = it->second;
  }
  if (placed) {
    // what each pending pod adds once assumed, as a bound pod's class: the bound pods' loop above from the other side
    std::map<std::vector<std::tuple<uint32_t, int32_t, uint8_t>>, uint32_t> qclass_of;
    pk.placed_class.assign(P, BS_IPF_NONE);
    for (size_t p = 0; p < P; ++p) {
      if (!pending[p]) continue;
      const Pod& pod = *pending[p];
      std::map<uint32_t, std::pair<int32_t, uint8_t>> ent;   // term -> (own, match)
      for (uint32_t id : own_anti[p]) ent[id].first = 1;
      for (auto& e : existing)
        if (pod_matches_term(pod, e.first)) ent[e.second].second = 1;
      for (const Set& s : sets) {
        bool all = true;
        for (const ResolvedTerm& r : s.terms) all = all && pod_matches_term(pod, r);
        if (all)
          for (uint32_t id : s.ids) ent[id].second = 1;
      }
      for (auto& a : antis)
        if (pod_matches_term(pod, a.first)) ent[a.second].second = 1;
      if (ent.empty()) continue;
      if (ent.size() > BS_IPF_CLASS_MAX)
        return Status{BS_CODE_ERROR, "PackInterPodFilter: a pending pod's placed class lists more than BS_IPF_CLASS_MAX terms"};
      std::vector<std::tuple<uint32_t, int32_t, uint8_t>> key;
      for (auto& kv : ent) key.emplace_back(kv.first, kv.second.first, kv.second.second);
      auto it = qclass_of.find(key);
      if (it == qclass_of.end()) {
        PackedInterPodAffinity::Classes& cl = pk.placed_classes;
        it = qclass_of.emplace(key, cl.n_classes()).first;
        for (auto& e : key) {
          cl.term.push_back(std::get<0>(e));
          cl.own.push_back(std::get<1>(e));
          cl.match.push_back(std::get<2>(e));
        }
        cl.offset.push_back((uint32_t)cl.term.size());
      }
      pk.placed_class[p] = it->second;
    }
  }
  number_topology(snapshot, pk.keys, &pk.values, &pk.n_values, &pk.topo);
  return Status{};
}

Status BatchSchedulingPlugin::UploadInterPodFilter() {
  auto fail = [&](int rc) {
    return Status{BS_CODE_ERROR, std::string("bsched: ") + bs_strerror(rc) + " (" + bs_last_error(eng_) + ")"};
  };
  int rc = bs_set_interpod_filter(eng_, interpod_filter_ ? 1 : 0);
  if (rc) return fail(rc);
  if (!interpod_filter_) return Status{};
  PackedInterPodFilter pk;
  Status st = PackInterPodFilter(snapshot_, pending_, &pk, interpod_filter_walks_);
  if (!st.ok()) return st;
  const PackedInterPodAffinity::Classes& c = pk.bound_classes;
  bs_interpod_nodes nt{(uint32_t)snapshot_.size(), (uint32_t)pk.keys.size(), pk.n_values.data(), pk.topo.data(),
                       (uint32_t)pk.term_key.size(), pk.term_key.data(), (uint32_t)pk.bound_node.size(),
                       pk.bound_node.data(), pk.bound_class.data(),
                       bs_interpod_classes{c.n_classes(), c.offset.data(), c.term.data(), c.own.data(), c.match.data()}};
  rc = bs_upload_node_interpod_filter(eng_, &nt);
  if (!rc) {
    bs_interpod_filter_pods pt{(uint32_t)pending_.size(), pk.pod_class.data(), pk.n_pod_classes(), pk.pod_offset.data(),
                               pk.pod_term.data(), pk.pod_role.data(), pk.self_match.data()};
    rc = bs_upload_pod_interpod_filter(eng_, &pt);
  }
  if (!rc && interpod_filter_walks_) {
    const PackedInterPodAffinity::Classes& q = pk.placed_classes;
    bs_interpod_pods qt{(uint32_t)pending_.size(), pk.placed_class.data(),
                        bs_interpod_classes{q.n_classes(), q.offset.data(), q.term.data(), q.own.data(), q.match.data()}};
    rc = bs_upload_pod_interpod_placed(eng_, &qt);
  }
  return rc ? fail(rc) : Status{};
}

void BatchSchedulingPlugin::SetHostPortFilter(bool on) {
  std::lock_guard<std::mutex> lk(mu_);
  host_port_filter_ = on;
}

void BatchSchedulingPlugin::SetHostPortFilterInPreemption(bool on) {
  std::lock_guard<std::mutex> lk(mu_);
  host_port_preempt_ = on;
}

namespace {
struct HostPortTriple {
  std::string ip, protocol;
  int32_t port;
  bool operator==(const HostPortTriple& o) const { return port == o.port && ip == o.ip && protocol == o.protocol; }
};
// HostPortInfo's sanitizing: port <= 0 is not a host port, "" ip is "0.0.0.0", "" protocol is "TCP"
void add_triples(const std::vector<ContainerPort>& ports, std::vector<HostPortTriple>* out) {
  for (const ContainerPort& cp : ports) {
    if (cp.host_port <= 0) continue;
    HostPortTriple t{cp.host_ip.empty() ? "0.0.0.0" : cp.host_ip, cp.protocol.empty() ? "TCP" : cp.protocol,
                     cp.host_port};
    if (std::find(out->begin(), out->end(), t) == out->end()) out->push_back(t);
  }
}
bool triples_conflict(const HostPortTriple& a, const HostPortTriple& b) {
  return a.protocol == b.protocol && a.port == b.port && (a.ip == "0.0.0.0" || b.ip == "0.0.0.0" || a.ip == b.ip);
}
}  // namespace

Status BatchSchedulingPlugin::PackHostPorts(const std::vector<const NodeInfo*>& snapshot,
                                            const std::vector<const Pod*>& pending, PackedHostPorts* out, bool bound) {
  if (!out) return Status{BS_CODE_ERROR, "PackHostPorts: null output"};
  *out = PackedHostPorts{};
  std::vector<HostPortTriple> dict;
  std::vector<std::vector<HostPortTriple>> wanted(pending.size()), used(snapshot.size());
  for (size_t p = 0; p < pending.size(); ++p) {
    if (pending[p])
      for (const Container& c : pending[p]->containers) add_triples(c.ports, &wanted[p]);
    for (const HostPortTriple& t : wanted[p])
      if (std::find(dict.begin(), dict.end(), t) == dict.end()) dict.push_back(t);
  }
  const size_t n_wanted = dict.size();
  for (size_t n = 0; n < snapshot.size(); ++n) {
    if (snapshot[n]) add_triples(snapshot[n]->used_ports, &used[n]);
    for (const HostPortTriple& t : used[n]) {
      if (std::find(dict.begin(), dict.end(), t) != dict.end()) continue;
      for (size_t k = 0; k < n_wanted; ++k)
        if (triples_conflict(dict[k], t)) {
          dict.push_back(t);
          break;
        }
    }
  }
  if (dict.size() > BS_HOSTPORT_MAX)
    return Status{BS_CODE_ERROR, "PackHostPorts: " + std::to_string(dict.size()) + " host-port entries, more than BS_HOSTPORT_MAX"};
  auto id = [](std::vector<std::string>& names, const std::string& s) {
    const auto it = std::find(names.begin(), names.end(), s);
    if (it != names.end()) return (uint32_t)(it - names.begin());
    names.push_back(s);
    return (uint32_t)names.size() - 1;
  };
  for (const HostPortTriple& t : dict) {
    out->ip.push_back(id(out->ips, t.ip));
    out->protocol.push_back(id(out->protocols, t.protocol));
    out->port.push_back(t.port);
  }
  auto mask = [&dict](const std::vector<HostPortTriple>& ts) {
    uint64_t m = 0;
    for (const HostPortTriple& t : ts) {
      const auto it = std::find(dict.begin(), dict.end(), t);
      if (it != dict.end()) m |= 1ull << (it - dict.begin());
    }
    return m;
  };
  for (const auto& ts : used) out->used.push_back(mask(ts));
  for (const auto& ts : wanted) out->want.push_back(mask(ts));
  if (bound) {   // PackBoundPods' rows: the snapshot's NodeInfo::pods in order
    std::vector<HostPortTriple> held;
    for (const NodeInfo* ni : snapshot)
      if (ni)
        for (const Pod* p : ni->pods) {
          if (!p) continue;
          held.clear();
          for (const Container& c : p->containers) add_triples(c.ports, &held);
          out->bound.push_back(mask(held));
        }
  }
  return Status{};
}

Status BatchSchedulingPlugin::UploadHostPorts() {
  auto fail = [&](int rc) {
    return Status{BS_CODE_ERROR, std::string("bsched: ") + bs_strerror(rc) + " (" + bs_last_error(eng_) + ")"};
  };
  int rc = bs_set_host_port_filter(eng_, host_port_filter_ ? 1 : 0);
  if (rc) return fail(rc);
  if (!host_port_filter_) return Status{};
  PackedHostPorts pk;
  Status st = PackHostPorts(snapshot_, pending_, &pk);
  if (!st.ok()) return st;
  bs_host_port_nodes nt{(uint32_t)snapshot_.size(), (uint32_t)pk.port.size(), pk.ip.data(), pk.protocol.data(),
                        pk.port.data(), pk.used.data()};
  rc = bs_upload_node_host_ports(eng_, &nt);
  if (!rc) rc = bs_upload_pod_host_ports(eng_, (uint32_t)pending_.size(), pk.want.data());
  return rc ? fail(rc) : Status{};
}

// Called right after every bound-table upload.  PackHostPorts numbers the dictionary from snapshot_ and pending_ alone,
// so the masks agree with the node and pod sides UploadHostPorts uploads in the same round or UpdateNodes.
Status BatchSchedulingPlugin::UploadBoundHostPorts() {
  if (!host_port_filter_ || !host_port_preempt_ || !bound_.n) return Status{};
  PackedHostPorts pk;
  Status st = PackHostPorts(snapshot_, pending_, &pk, true);
  if (!st.ok()) return st;
  const int rc = bs_upload_bound_host_ports(eng_, (uint32_t)pk.bound.size(), pk.bound.data());
  if (rc) return Status{BS_CODE_ERROR, std::string("bsched: ") + bs_strerror(rc) + " (" + bs_last_error(eng_) + ")"};
  return Status{};
}

std::vector<uint32_t> BatchSchedulingPlugin::HostPortReasonCounts(const std::string& uid) const {
  const int32_t row = pod_row_.find(uid);
  if (row < 0 || hp_reasons_.size() <= (size_t)row) return {};
  return {hp_reasons_[row]};
}

std::vector<uint32_t> BatchSchedulingPlugin::InterPodReasonCounts(const std::string& uid) const {
  const int32_t row = pod_row_.find(uid);
  if (row < 0 || ipf_reasons_.size() < ((size_t)row + 1) * 3) return {};
  return std::vector<uint32_t>(ipf_reasons_.begin() + (size_t)row * 3, ipf_reasons_.begin() + ((size_t)row + 1) * 3);
}

Status BatchSchedulingPlugin::UploadInterPodAffinity() {
  if (!priority_k_) return Status{};
  auto fail = [&](int rc) {
    return Status{BS_CODE_ERROR, std::string("bsched: ") + bs_strerror(rc) + " (" + bs_last_error(eng_) + ")"};
  };
  int rc = bs_set_interpod_weight(eng_, interpod_weight_);
  if (rc) return fail(rc);
  if (!interpod_weight_) return Status{};
  PackedInterPodAffinity pk;
  Status st = PackInterPodAffinity(snapshot_, pending_, hard_pod_affinity_weight_, &pk);
  if (!st.ok()) return st;
  auto classes = [](const PackedInterPodAffinity::Classes& c) {
    return bs_interpod_classes{c.n_classes(), c.offset.data(), c.term.data(), c.own.data(), c.match.data()};
  };
  bs_interpod_nodes nt{(uint32_t)snapshot_.size(), (uint32_t)pk.keys.size(), pk.n_values.data(), pk.topo.data(),
                       (uint32_t)pk.term_key.size(), pk.term_key.data(), (uint32_t)pk.bound_node.size(),
                       pk.bound_node.data(), pk.bound_class.data(), classes(pk.bound_classes)};
  rc = bs_upload_node_interpod(eng_, &nt);
  if (!rc) {
    bs_interpod_pods pt{(uint32_t)pending_.size(), pk.pod_class.data(), classes(pk.pod_classes)};
    rc = bs_upload_pod_interpod(eng_, &pt);
  }
  return rc ? fail(rc) : Status{};
}

std::vector<uint32_t> BatchSchedulingPlugin::ReasonCounts(const std::string& uid) const {
  const int32_t row = pod_row_.find(uid);
  const size_t R = 4 + packed_.lanes;
  if (row < 0 || reasons_.size() < ((size_t)row + 1) * R) return {};
  return std::vector<uint32_t>(reasons_.begin() + (size_t)row * R, reasons_.begin() + ((size_t)row + 1) * R);
}

std::string BatchSchedulingPlugin::FitError(const std::string& uid) const {
  const int32_t row = pod_row_.find(uid);
  if (row < 0 || (size_t)row >= feasible_.size() || feasible_[row] != 0) return "";
  const std::vector<uint32_t> counts = ReasonCounts(uid);
  if (counts.empty()) return "";
  std::vector<const char*> names;
  for (auto& nm : packed_.scalar_names) names.push_back(nm.c_str());
  const std::vector<uint32_t> ipf = InterPodReasonCounts(uid);   // empty while the filter is off
  const std::vector<uint32_t> hp = HostPortReasonCounts(uid);     // likewise
  std::vector<char> buf(256);
  for (;;) {   // grows until the whole message fits
    const int rc = bs_format_fit_error_filters(counts.data(), packed_.lanes, ipf.empty() ? nullptr : ipf.data(),
                                               hp.empty() ? nullptr : hp.data(), packed_.n_nodes,
                                               names.empty() ? nullptr : names.data(), buf.data(), buf.size());
    if (rc == BS_OK) return std::string(buf.data());
    if (buf.size() > (1u << 20)) return "";
    buf.resize(buf.size() * 4);
  }
}

Status BatchSchedulingPlugin::UpdateRound(const std::vector<std::pair<uint32_t, const NodeInfo*>>& changed_nodes,
                                          const std::vector<std::string>& changed_groups, int64_t now_ns) {
  if (!eng_) return Status{BS_CODE_ERROR, "UpdateRound: no round has been started"};
  now_ns_ = now_ns;
  Status st = UpdateNodes(changed_nodes, false);
  if (!st.ok()) return st;
  st = UpdateGroups(changed_groups, now_ns, false);
  if (!st.ok()) return st;
  if (changed_nodes.empty()) {   // UpdateNodes uploaded the preferences and weights when it changed rows
    st = UploadPreferences();
    if (!st.ok()) return st;
    st = UploadLocality();
    if (!st.ok()) return st;
    st = UploadSpread();
    if (!st.ok()) return st;
    st = UploadInterPodAffinity();
    if (!st.ok()) return st;
    st = UploadInterPodFilter();
    if (!st.ok()) return st;
    st = UploadHostPorts();
    if (!st.ok()) return st;
  }
  return Reevaluate();
}

Status BatchSchedulingPlugin::UpdateNodes(const std::vector<std::pair<uint32_t, const NodeInfo*>>& changed, bool evaluate) {
  if (!eng_) return Status{BS_CODE_ERROR, "UpdateNodes: no round has been started"};
  if (changed.empty()) return Status{};
  std::vector<const NodeInfo*> rows(changed.size());
  std::vector<uint32_t> idx(changed.size());
  for (size_t k = 0; k < changed.size(); ++k) {
    if (changed[k].first >= packed_.n_nodes) return Status{BS_CODE_ERROR, "UpdateNodes: index outside the snapshot"};
    idx[k] = changed[k].first;
    rows[k] = changed[k].second;
  }
  PackedSnapshot delta;
  bool needs_full = false;
  Status st = PackNodeRows(packed_, rows, &delta, &needs_full);
  if (!st.ok()) return st;
  if (needs_full) return Status{BS_CODE_ERROR, "full repack needed"};
  bs_node_table t = delta.node_table();
  int rc = bs_update_nodes(eng_, idx.data(), &t);
  if (rc) return Status{BS_CODE_ERROR, std::string("bsched: ") + bs_strerror(rc) + " (" + bs_last_error(eng_) + ")"};
  if (packed_.n_aff()) {   // the changed nodes' labels may have moved their affinity verdicts
    const uint32_t W = (packed_.n_nodes + 31) / 32, nrow = delta.n_nodes;
    for (uint32_t c = 0; c < packed_.n_aff(); ++c)
      for (uint32_t k = 0; k < nrow; ++k) {
        uint32_t& word = packed_.aff_bits[(size_t)c * W + (idx[k] >> 5)];
        const uint32_t bit = 1u << (idx[k] & 31);
        word = delta.aff_bits[(size_t)c * nrow + k] ? (word | bit) : (word & ~bit);
      }
    rc = bs_upload_affinity(eng_, packed_.n_aff(), packed_.aff_bits.data());
    if (rc) return Status{BS_CODE_ERROR, std::string("bsched: ") + bs_strerror(rc) + " (" + bs_last_error(eng_) + ")"};
  }
  // keep the host copy of the round in step with the device table
  const uint32_t N = packed_.n_nodes, n = delta.n_nodes, L = packed_.lanes;
  for (uint32_t k = 0; k < n; ++k) {
    const uint32_t i = idx[k];
    for (uint32_t d = 0; d < L; ++d) {
      packed_.alloc[(size_t)d * N + i] = delta.alloc[(size_t)d * n + k];
      packed_.requested[(size_t)d * N + i] = delta.requested[(size_t)d * n + k];
    }
    packed_.pod_count[i] = delta.pod_count[k]; packed_.alloc_present[i] = delta.alloc_present[k];
    packed_.req_present[i] = delta.req_present[k]; packed_.label_mask[i] = delta.label_mask[k];
    packed_.taint_mask[i] = delta.taint_mask[k]; packed_.node_flags[i] = delta.node_flags[k];
    if (i < snapshot_.size()) snapshot_[i] = rows[k];
  }
  st = UploadBound();   // bs_update_nodes dropped the bound-pod table: the changed NodeInfos list their pods again
  if (!st.ok()) return st;
  st = UploadNonZero(nullptr);   // ... and the node non-zero column: the changed NodeInfos' pods count again
  if (!st.ok()) return st;
  st = UploadPreferences();      // ... and the node preference side (its taint dictionary may change: both sides)
  if (!st.ok()) return st;
  st = UploadLocality();         // ... and the locality side (its dictionaries may change: both sides)
  if (!st.ok()) return st;
  st = UploadSpread();           // ... and the spread side (the changed NodeInfos' pods and zones: both sides)
  if (!st.ok()) return st;
  st = UploadInterPodAffinity();   // ... and the inter-pod side (the changed NodeInfos' pods and labels: both sides)
  if (!st.ok()) return st;
  st = UploadInterPodFilter();     // ... and the filter's sides, for the same reasons
  if (!st.ok()) return st;
  st = UploadHostPorts();          // ... and the host-port sides (the changed NodeInfos' used ports)
  if (!st.ok()) return st;
  // the round's decisions follow the new snapshot: same pods, same groups, same result vectors
  return evaluate ? Reevaluate() : Status{};
}

Status BatchSchedulingPlugin::PackGroupRows(const PackedSnapshot& ctx, const std::vector<GroupDelta>& rows,
                                            int64_t default_wait_ns, PackedSnapshot* out, bool* needs_full) {
  if (!out || !needs_full) return Status{BS_CODE_ERROR, "PackGroupRows: null output"};
  *needs_full = false;
  PackedSnapshot& ps = *out;
  ps = PackedSnapshot();
  const uint32_t n = (uint32_t)rows.size();
  ps.lanes = ctx.lanes; ps.scalar_names = ctx.scalar_names; ps.sel_pairs = ctx.sel_pairs; ps.taint_list = ctx.taint_list;
  ps.n_groups = n;
  const RowEncoder enc(ctx, ps);
  for (uint32_t k = 0; k < n; ++k) {
    const GroupDelta& gd = rows[k];
    if (!gd.pg || gd.index >= ctx.n_groups) return Status{BS_CODE_ERROR, "PackGroupRows: bad row"};
    ps.name_rank[k] = ctx.name_rank[gd.index];   // the name of an object does not change
    const Encoded r = enc.group(gd, k, n, default_wait_ns);
    if (r == kNeedsFull) { *needs_full = true; return Status{}; }
    if (r != kEncoded) return Status{BS_CODE_ERROR, kEncodeError[r]};
  }
  return Status{};
}

Status BatchSchedulingPlugin::UpdateGroups(const std::vector<std::string>& ns_names, int64_t now_ns, bool evaluate) {
  if (!eng_) return Status{BS_CODE_ERROR, "UpdateGroups: no round has been started"};
  if (ns_names.empty()) return Status{};
  now_ns_ = now_ns;
  std::vector<GroupDelta> rows;
  std::vector<uint32_t> idx;
  for (auto& name : ns_names) {
    const int gi = group_index(name);
    auto it = groups_.find(name);
    if (gi < 0 || it == groups_.end()) return Status{BS_CODE_ERROR, "UpdateGroups: " + name + " is not part of the round (full repack needed)"};
    GroupState& gs = it->second;
    uint32_t matched = 0;
    int32_t sched = 0, den = 0;
    bs_group_state(eng_, (uint32_t)gi, now_ns, &matched, &sched, &den);
    uint8_t fl = 0;
    if (sched) fl |= BS_GROUP_SCHEDULED;
    if (den) fl |= BS_GROUP_DENIED;
    GroupDelta gd;
    gd.index = (uint32_t)gi; gd.pg = &gs.pg; gd.matched = matched; gd.flags = fl;
    gd.rep_pod = gs.has_pod ? &gs.rep_pod : nullptr;
    rows.push_back(gd);
    idx.push_back((uint32_t)gi);
  }
  PackedSnapshot delta;
  bool needs_full = false;
  Status st = PackGroupRows(packed_, rows, max_schedule_time_ns_, &delta, &needs_full);
  if (!st.ok()) return st;
  if (needs_full) return Status{BS_CODE_ERROR, "full repack needed"};
  bs_group_table t = delta.group_table();
  int rc = bs_update_groups(eng_, idx.data(), &t);
  if (rc) return Status{BS_CODE_ERROR, std::string("bsched: ") + bs_strerror(rc) + " (" + bs_last_error(eng_) + ")"};
  const uint32_t G = packed_.n_groups, n = delta.n_groups, L = packed_.lanes;
  for (uint32_t k = 0; k < n; ++k) {
    const uint32_t g = idx[k];
    packed_.min_member[g] = delta.min_member[k]; packed_.scheduled[g] = delta.scheduled[k];
    packed_.matched[g] = delta.matched[k]; packed_.group_flags[g] = delta.group_flags[k];
    for (uint32_t d = 0; d < L; ++d) packed_.min_res[(size_t)d * G + g] = delta.min_res[(size_t)d * n + k];
    packed_.min_res_present[g] = delta.min_res_present[k]; packed_.rep_sel[g] = delta.rep_sel[k];
    packed_.rep_tol[g] = delta.rep_tol[k]; packed_.creation_ns[g] = delta.creation_ns[k];
    if (packed_.rep_aff.size() == G) packed_.rep_aff[g] = delta.rep_aff[k];
    packed_.wait_ns[g] = delta.wait_ns[k];
  }
  if ((rc = bs_set_wait_time(eng_, max_schedule_time_ns_, packed_.wait_ns.data(), G)))
    return Status{BS_CODE_ERROR, std::string("bsched: ") + bs_strerror(rc)};
  st = UploadBound();   // a changed Status.Phase locks or unlocks the bound pods of its group
  if (!st.ok()) return st;
  return evaluate ? Reevaluate() : Status{};
}

// ---- preemption: the bound-pod table, RemovePod, Preempt ----
bs_bound_table PackedBound::table() const {
  return bs_bound_table{n, lanes, node.data(), req.data(), req_present.data(), gid.data(), priority.data(),
                        start_ns.data(), flags.data()};
}

Status BatchSchedulingPlugin::PackBoundPods(const PackedSnapshot& ctx, const std::vector<const NodeInfo*>& snapshot,
                                            const std::unordered_map<std::string, uint32_t>& group_row,
                                            const std::vector<uint8_t>& locked, PackedBound* out,
                                            const std::vector<PodDisruptionBudget>& pdbs) {
  if (!out) return Status{BS_CODE_ERROR, "PackBoundPods: null output"};
  // filterPodsWithPDBViolation: only a budget that allows no disruption can make a pod violating; its selector is
  // converted once here.  A nil or empty selector matches nothing, and one that fails to convert is skipped.
  std::vector<std::pair<const std::string*, SpreadSel>> exhausted;
  for (const PodDisruptionBudget& pdb : pdbs) {
    SpreadSel sel;
    if (pdb.disruptions_allowed > 0 || !pdb.has_selector || !sel_from_label_selector(pdb.selector, &sel) || sel.empty())
      continue;
    exhausted.emplace_back(&pdb.ns, std::move(sel));
  }
  PackedBound& b = *out;
  b = PackedBound();
  b.lanes = ctx.lanes;
  LaneTable lt;
  for (auto& s : ctx.scalar_names) lt.add(s);   // lane 4 + k, as in the round
  for (uint32_t i = 0; i < snapshot.size(); ++i)
    if (snapshot[i])
      for (const Pod* p : snapshot[i]->pods)
        if (p) b.pods.push_back(p), b.node.push_back(i);
  const uint32_t V = b.n = (uint32_t)b.pods.size(), L = b.lanes;
  b.req.assign((size_t)L * V, 0);
  b.req_present.assign(V, 0); b.gid.assign(V, BS_GID_NONE); b.priority.assign(V, 0); b.start_ns.assign(V, 0);
  b.flags.assign(V, 0);
  std::vector<int64_t> v(L);
  for (uint32_t k = 0; k < V; ++k) {
    const Pod& p = *b.pods[k];
    std::fill(v.begin(), v.end(), 0);
    for (const Container& c : p.containers) {
      // NodeInfo.RemovePod subtracts the pod's Requests (calculateResource, [upstream, from memory]), never its Limits
      const Encoded r = add_list(lt, c.requests, v.data(), &b.req_present[k], kBadContainers);
      if (r == kNeedsFull)
        return Status{BS_CODE_ERROR, "PackBoundPods: pod " + p.ns + "/" + p.name + " requests a scalar resource its node's requested lacks"};
      if (r != kEncoded) return Status{BS_CODE_ERROR, std::string("PackBoundPods: ") + kEncodeError[r]};
    }
    for (uint32_t d = 0; d < L; ++d) b.req[(size_t)d * V + k] = d == (uint32_t)kLanePods ? 0 : v[d];
    b.priority[k] = p.priority;
    b.start_ns[k] = p.start_ns;
    auto lb = p.labels.find(kPodGroupLabel);   // VerifyPodLabelSatisfied (k8s.go:62-70)
    if (lb != p.labels.end() && !lb->second.empty()) {
      auto it = group_row.find(p.ns + "/" + lb->second);   // checkPreemption's fullNameToRemove (core.go:221)
      if (it == group_row.end()) b.gid[k] = BS_GID_MISSING;
      else {
        b.gid[k] = (int32_t)it->second;
        if (it->second < locked.size() && locked[it->second]) b.flags[k] = BS_BOUND_GROUP_LOCKED;
      }
    }
    if (!p.labels.empty())   // a pod without labels matches no budget
      for (const auto& e : exhausted)
        if (*e.first == p.ns && spread_sel_matches(e.second, p.labels)) {
          b.flags[k] |= BS_BOUND_PDB_VIOLATING;
          break;
        }
  }
  return Status{};
}

Status BatchSchedulingPlugin::UploadBound() {
  bool any = false;
  for (const NodeInfo* ni : snapshot_) any = any || (ni && !ni->pods.empty());
  if (!any) {
    bound_ = PackedBound();
    bound_row_.clear();
    return Status{};
  }
  std::vector<uint8_t> locked(group_names_.size(), 0);
  for (size_t g = 0; g < group_names_.size(); ++g) {
    auto it = groups_.find(group_names_[g]);
    if (it != groups_.end()) locked[g] = it->second.pg.phase == "Scheduled" || it->second.pg.phase == "Running";
  }
  Status st = PackBoundPods(packed_, snapshot_, group_row_, locked, &bound_, pdbs_);
  if (!st.ok()) return st;
  bound_row_.build(bound_.n, [&](size_t k) { return &bound_.pods[k]->uid; }, pack_threads(bound_.n));
  const bs_bound_table t = bound_.table();
  const int rc = bs_upload_bound_pods(eng_, &t);
  if (rc) return Status{BS_CODE_ERROR, std::string("bsched: ") + bs_strerror(rc) + " (" + bs_last_error(eng_) + ")"};
  return UploadBoundHostPorts();   // the masks belong to the table just uploaded
}

Status BatchSchedulingPlugin::RemovePod(const Pod& preemptor, const Pod& victim) {
  std::lock_guard<std::mutex> lk(mu_);
  const int32_t p = pod_row_.find(preemptor.uid), v = bound_row_.find(victim.uid);
  if (!eng_ || p < 0 || v < 0) return Status{BS_CODE_ERROR, "RemovePod: the pods are not part of the round"};
  bs_status st{};
  int rc = bs_remove_pod(eng_, (uint32_t)p, (uint32_t)v, &st);
  if (rc) return Status{BS_CODE_ERROR, std::string("bsched: ") + bs_strerror(rc) + " (" + bs_last_error(eng_) + ")"};
  if (st.code == BS_CODE_SUCCESS) return Status{};
  auto lb = victim.labels.find(kPodGroupLabel);
  const std::string victim_group = victim.ns + "/" + (lb == victim.labels.end() ? std::string() : lb->second);
  char buf[1024];
  rc = bs_format_remove_message(&st, preemptor.name.c_str(), victim.name.c_str(), victim_group.c_str(), buf, sizeof buf);
  if (rc) return Status{BS_CODE_ERROR, "RemovePod: message does not fit"};
  return Status{st.code, buf};   // framework.NewStatus(framework.Unschedulable, err.Error()) (batchscheduler.go:137-141)
}

Status BatchSchedulingPlugin::RunPreempt(const std::vector<uint32_t>& rows, std::vector<Preemption>* out,
                                         int walk_flags) {
  const uint32_t n = (uint32_t)rows.size();
  std::vector<int32_t> node(n);
  std::vector<uint32_t> nv(n), cand(n), off(n + 1);
  std::vector<uint32_t> vict;
  bs_preempt_result r{node.data(), nv.data(), cand.data(), off.data(), nullptr, 0, 0};
  auto call = [&] {
    return walk_flags < 0 ? bs_preempt(eng_, rows.data(), n, &r)
                          : bs_preempt_walk(eng_, rows.data(), n, (uint32_t)walk_flags, &r, nullptr, nullptr);
  };
  int rc = call();
  if (rc == BS_E_INVAL && r.victims_total > 0) {   // the first call sized the victim list
    vict.resize(r.victims_total);
    r.victims = vict.data();
    r.victims_cap = r.victims_total;
    rc = call();
  }
  if (rc) return Status{BS_CODE_ERROR, std::string("bsched: ") + bs_strerror(rc) + " (" + bs_last_error(eng_) + ")"};
  out->resize(n);
  for (uint32_t i = 0; i < n; ++i) {
    Preemption& pr = (*out)[i];
    pr.node = node[i] >= 0 ? node_names_[node[i]] : std::string();
    pr.victims.clear();
    for (uint32_t k = off[i]; k < off[i + 1]; ++k) pr.victims.push_back(bound_.pods[vict[k]]->uid);
  }
  return Status{};
}

Status BatchSchedulingPlugin::Preempt(const std::string& uid, std::string* node, std::vector<std::string>* victim_uids) {
  std::lock_guard<std::mutex> lk(mu_);
  if (interpod_filter_)
    return Status{BS_CODE_ERROR, "Preempt: the MatchInterPodAffinity filter is on (SetInterPodAffinityFilter(false) first)"};
  if (host_port_filter_ && !host_port_preempt_)
    return Status{BS_CODE_ERROR, "Preempt: the PodFitsHostPorts filter is on (SetHostPortFilter(false) first)"};
  const int32_t p = pod_row_.find(uid);
  if (!eng_ || p < 0) return Status{BS_CODE_ERROR, "Preempt: " + uid + " is not a pending pod of the round"};
  if (!bound_.n) {   // no NodeInfo lists pods: nothing to evict, the table was never uploaded
    if (node) node->clear();
    if (victim_uids) victim_uids->clear();
    return Status{};
  }
  std::vector<Preemption> res;
  Status st = RunPreempt({(uint32_t)p}, &res);
  if (!st.ok()) return st;
  if (node) *node = res[0].node;
  if (victim_uids) *victim_uids = res[0].victims;
  return Status{};
}

Status BatchSchedulingPlugin::PreemptAll(std::vector<Preemption>* out) {
  std::lock_guard<std::mutex> lk(mu_);
  if (!eng_ || !out) return Status{BS_CODE_ERROR, "PreemptAll: no round has been started"};
  if (interpod_filter_)
    return Status{BS_CODE_ERROR, "PreemptAll: the MatchInterPodAffinity filter is on (SetInterPodAffinityFilter(false) first)"};
  if (host_port_filter_ && !host_port_preempt_)
    return Status{BS_CODE_ERROR, "PreemptAll: the PodFitsHostPorts filter is on (SetHostPortFilter(false) first)"};
  out->clear();
  if (!bound_.n) return Status{};
  std::vector<uint32_t> rows;
  for (uint32_t i = 0; i < packed_.n_pods; ++i)
    if (prefilter_[i] == BS_PF_PASS && feasible_[i] == 0) rows.push_back(i);
  if (rows.empty()) return Status{};
  Status st = RunPreempt(rows, out);
  if (!st.ok()) return st;
  for (size_t k = 0; k < rows.size(); ++k) (*out)[k].uid = pending_uid_[rows[k]];
  return Status{};
}

Status BatchSchedulingPlugin::PreemptQueue(std::vector<Preemption>* out, bool gang) {
  std::lock_guard<std::mutex> lk(mu_);
  if (!eng_ || !out) return Status{BS_CODE_ERROR, "PreemptQueue: no round has been started"};
  if (interpod_filter_)
    return Status{BS_CODE_ERROR, "PreemptQueue: the MatchInterPodAffinity filter is on (SetInterPodAffinityFilter(false) first)"};
  if (host_port_filter_ && !host_port_preempt_)
    return Status{BS_CODE_ERROR, "PreemptQueue: the PodFitsHostPorts filter is on (SetHostPortFilter(false) first)"};
  out->clear();
  if (!bound_.n) return Status{};
  // PreemptAll's pods in queue order; with gang units, one unit per group at its first preemptor's place
  std::vector<std::vector<uint32_t>> units;
  std::unordered_map<int32_t, size_t> unit_of;
  for (uint32_t i : order_) {
    if (prefilter_[i] != BS_PF_PASS || feasible_[i] != 0) continue;
    const int32_t g = packed_.gid[i];
    if (gang && g >= 0) {
      auto it = unit_of.find(g);
      if (it != unit_of.end()) {
        std::vector<uint32_t>& u = units[it->second];
        if (packed_.priority[i] != packed_.priority[u[0]])
          return Status{BS_CODE_ERROR, "PreemptQueue: the pending pods of group " + group_names_[g] +
                                           " have different priorities"};
        u.push_back(i);
        continue;
      }
      unit_of[g] = units.size();
    }
    units.push_back({i});
  }
  std::vector<uint32_t> rows;
  for (const std::vector<uint32_t>& u : units) rows.insert(rows.end(), u.begin(), u.end());
  if (rows.empty()) return Status{};
  Status st = RunPreempt(rows, out, gang ? (int)BS_PREEMPT_GANG : 0);
  if (!st.ok()) return st;
  for (size_t k = 0; k < rows.size(); ++k) (*out)[k].uid = pending_uid_[rows[k]];
  return Status{};
}

Status BatchSchedulingPlugin::ReplayQueue(std::vector<ReplayDecision>* out, ReplayNodeChoice choice) {
  if (!out) return Status{BS_CODE_ERROR, "ReplayQueue: null output"};
  if (!eng_) return Status{BS_CODE_ERROR, "ReplayQueue: no round has been started"};
  if (interpod_filter_ && !interpod_filter_walks_)
    return Status{BS_CODE_ERROR, "ReplayQueue: the MatchInterPodAffinity filter is on (SetInterPodAffinityFilter(false) first)"};
  const bool prio = choice == ReplayNodeChoice::kPriority;
  if (prio && !priority_k_)
    return Status{BS_CODE_ERROR, "ReplayQueue: kPriority needs a plugin created with priority_k > 0 (its rounds upload "
                                 "the non-zero request columns)"};
  if (prio && (node_prio_weights_[0] || node_prio_weights_[1]))
    return Status{BS_CODE_ERROR, "ReplayQueue: kPriority does not support TaintToleration and NodeAffinity yet "
                                 "(SetNodePriorityWeights(0, 0) first)"};
  if (prio && spread_weight_)
    return Status{BS_CODE_ERROR, "ReplayQueue: kPriority does not support SelectorSpread yet "
                                 "(SetSelectorSpreadWeight(0) first)"};
  if (prio && interpod_weight_)
    return Status{BS_CODE_ERROR, "ReplayQueue: kPriority does not support InterPodAffinity yet "
                                 "(SetInterPodAffinityWeight(0) first)"};
  const uint32_t P = packed_.n_pods;
  std::vector<uint8_t> pf(P), rd(P);
  std::vector<int32_t> nd(P);
  bs_replay_result r{};
  r.prefilter = pf.data(); r.node = nd.data(); r.ready = rd.data();
  const int rc = prio ? bs_replay_priority(eng_, order_.data(), P, &r, nullptr) : bs_replay(eng_, order_.data(), P, &r);
  if (rc) return Status{BS_CODE_ERROR, std::string("bsched: ") + bs_strerror(rc) + " (" + bs_last_error(eng_) + ")"};
  out->assign(P, ReplayDecision{});
  for (uint32_t qi = 0; qi < P; ++qi) (*out)[order_[qi]] = ReplayDecision{pf[qi], nd[qi], rd[qi] != 0, qi};
  return Status{};
}

Status BatchSchedulingPlugin::PreFilter(const Pod& pod) {
  const int32_t row = pod_row_.find(pod.uid);
  if (row < 0) return Status{BS_CODE_ERROR, "pod is not part of the current round"};
  bs_status st{};
  int rc = bs_prefilter(eng_, (uint32_t)row, &st);
  if (rc) return Status{BS_CODE_ERROR, bs_strerror(rc)};
  if (st.reason == BS_PF_PASS) return Status{};                                 // batchscheduler.go:107
  std::string ns_name, occ;
  auto lab = pod.labels.find(kPodGroupLabel);
  if (lab != pod.labels.end()) ns_name = pod.ns + "/" + lab->second;            // fullName core.go:93
  if (st.group >= 0) occ = groups_[group_names_[st.group]].pg.occupied_by;
  char buf[512];
  bs_format_message(&st, ns_name.c_str(), occ.c_str(), buf, sizeof(buf));
  return Status{BS_CODE_UNSCHEDULABLE, buf};                                    // batchscheduler.go:104-106
}

std::pair<Status, int64_t> BatchSchedulingPlugin::Permit(const Pod& pod, const std::string& node_name,
                                                         bool* start_signal) {
  if (start_signal) *start_signal = false;
  int32_t row, nrow;
  {
    std::lock_guard<std::mutex> lk(mu_);
    row = pod_row_.find(pod.uid);
    nrow = node_row_.find(node_name);
    if (row < 0 || nrow < 0)
      return {Status{BS_CODE_ERROR, "pod or node is not part of the current round"}, 0};
  }
  bs_permit_result r{};
  // core.Permit with its bookkeeping (MatchedPodNodes.Set, the name -> uid de-dup of core.go:286-296, PodNameUIDs.Set,
  // ready on the live count, pgs.Scheduled) against the engine's TTL tables
  int rc = bs_permit_at(eng_, (uint32_t)row, (uint32_t)nrow, now_ns_, &r);
  if (rc) return {Status{BS_CODE_ERROR, bs_strerror(rc)}, 0};
  if (r.code == BS_CODE_UNSCHEDULABLE) {
    auto lab = pod.labels.find(kPodGroupLabel);
    return {Status{BS_CODE_UNSCHEDULABLE, "can not found pod group: " + (lab != pod.labels.end() ? lab->second : std::string())},
            r.wait_ns};                                                          // core.go:276, batchscheduler.go:194-195
  }
  if (r.group >= 0) {
    std::lock_guard<std::mutex> lk(mu_);
    uid_of_id_[IdOf(pod.uid)] = pod.uid;
  }
  if (start_signal) *start_signal = r.start_signal != 0;                         // batchscheduler.go:197-199
  return {Status{r.code, ""}, r.wait_ns};
}

Status BatchSchedulingPlugin::Filter(const Pod& pod, const std::string& node_name) {
  const int32_t row = pod_row_.find(pod.uid), nrow = node_row_.find(node_name);
  if (row < 0 || nrow < 0)
    return Status{BS_CODE_ERROR, "pod or node is not part of the current round"};
  bs_status st{};
  int rc = bs_filter(eng_, (uint32_t)row, (uint32_t)nrow, &st);
  if (rc) return Status{BS_CODE_ERROR, std::string("bsched: ") + bs_strerror(rc)};
  auto lab = pod.labels.find(kPodGroupLabel);
  const std::string pg_name = lab != pod.labels.end() ? lab->second : std::string();
  switch (st.reason) {
    case BS_FILTER_PASS:
      if (!pg_name.empty()) AddPermitted(pod.uid, now_ns_);                       // core.go:188
      return Status{};
    case BS_FILTER_ERR_NOT_FOUND:
      return Status{BS_CODE_UNSCHEDULABLE, "can not found pod group: " + pg_name};  // core.go:179 (bare name)
    case BS_FILTER_ERR_NO_SNAPSHOT:
      AddToDenyCache(pod.ns + "/" + pg_name, now_ns_);                            // core.go:184
      return Status{BS_CODE_UNSCHEDULABLE, "SnapShot not initialized"};           // core.go:547
    case BS_FILTER_ERR_NOT_ENOUGH:
      AddToDenyCache(pod.ns + "/" + pg_name, now_ns_);
      return Status{BS_CODE_UNSCHEDULABLE, "resource not enough"};                // util.ErrorResourceNotEnough
    default:
      return Status{BS_CODE_ERROR, "reference would dereference a nil maxPGStatus (core.go:525)"};
  }
}

// ScheduleOperation.Compare (core.go:368-411), from the two pods and the PodGroup cache alone — the scheduling
// queue calls Less at any time on any two pods, also ones no round has seen yet.
bool BatchSchedulingPlugin::Less(const Pod& a, const Pod& b) {
  std::lock_guard<std::mutex> lk(mu_);
  auto pg_name = [](const Pod& p) {                            // util.VerifyPodLabelSatisfied k8s.go:62-70
    auto it = p.labels.find(kPodGroupLabel);
    return it == p.labels.end() ? std::string() : it->second;
  };
  const std::string n1 = pg_name(a), n2 = pg_name(b);
  if (a.priority > b.priority) return true;                    // :380-382
  if (a.priority == b.priority) {
    if (n1.empty() && n2.empty()) return a.queue_ts_ns < b.queue_ts_ns;   // :385-387
    if (n1.empty()) return true;                               // :389-391
    if (n2.empty()) return false;                              // :392-394
  }
  auto g1 = groups_.find(a.ns + "/" + n1), g2 = groups_.find(b.ns + "/" + n2);   // pgLister.PodGroups(ns).Get(name) :395-396
  if (g1 == groups_.end() || g2 == groups_.end()) return false;                  // :397-399
  if (a.priority != b.priority) return false;
  const int64_t c1 = g1->second.pg.creation_ns, c2 = g2->second.pg.creation_ns;
  if (c1 < c2) return true;                                    // :400-402
  if (c1 == c2 && n1 > n2) return true;                        // :404-406
  return c1 == c2 && n1 == n2 && a.queue_ts_ns < b.queue_ts_ns;   // :407-408
}

}  // namespace bsched
