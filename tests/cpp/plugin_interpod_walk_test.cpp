// plugin_interpod_walk_test.cpp — BatchSchedulingPlugin::PackInterPodFilter's placed classes and
// SetInterPodAffinityFilterInWalks, printed as JSON for tests/test_plugin_interpod_walk.py.  Seeded rounds of ten roomy
// nodes (hostname, zone and rack keys, some nodes without the zone or rack key, one NodeInfo without a Node) with bound
// pods whose required anti-affinity terms and pending pods whose required affinity and anti-affinity terms use nil,
// empty, matchLabels and invalid selectors, listed and empty namespaces and an empty topology key; no pod belongs to a
// PodGroup.  The program prints the objects and the columns PackInterPodFilter made of them, without and with the
// placed side.  With the argument "gpu" it also runs each scenario through a plugin with SetInterPodAffinityFilter(true):
// whether ReplayQueue refuses without SetInterPodAffinityFilterInWalks, and with it the queue order and the nodes of
// ReplayQueue's first-fit and priority walks, and the first-fit walk again after UpdateNodes.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <string>
#include <vector>

#include "../../batch-scheduler_b200/csrc/plugin.hpp"

using namespace bsched;

static std::string q(const std::string& s) {
  std::string o = "\"";
  for (char c : s) {
    if (c == '"' || c == '\\') { o += '\\'; o += c; }
    else if ((unsigned char)c < 0x20) { char b[8]; snprintf(b, sizeof b, "\\u%04x", c); o += b; }
    else o += c;
  }
  return o + "\"";
}
static std::string jmap(const std::map<std::string, std::string>& m) {
  std::string o = "{";
  for (auto& kv : m) o += (o.size() > 1 ? ", " : "") + q(kv.first) + ": " + q(kv.second);
  return o + "}";
}
static std::string jstrs(const std::vector<std::string>& v) {
  std::string o = "[";
  for (size_t k = 0; k < v.size(); ++k) o += (k ? ", " : "") + q(v[k]);
  return o + "]";
}
// a selector as the object restatement reads it: null (nil), "invalid", or its match_labels
static std::string jterm(const PodAffinityTerm& t) {
  std::string sel = !t.has_selector ? "null" : !t.selector.match_expressions.empty() ? "\"invalid\"" : jmap(t.selector.match_labels);
  return "{\"selector\": " + sel + ", \"namespaces\": " + jstrs(t.namespaces) + ", \"key\": " + q(t.topology_key) + "}";
}
static std::string jterms(const std::vector<PodAffinityTerm>& v) {
  std::string o = "[";
  for (size_t k = 0; k < v.size(); ++k) o += (k ? ", " : "") + jterm(v[k]);
  return o + "]";
}
static std::string jpod(const Pod& p) {
  return "{\"name\": " + q(p.name) + ", \"ns\": " + q(p.ns) + ", \"labels\": " + jmap(p.labels) + ", \"terminating\": " +
         (p.terminating ? "true" : "false") + ", \"affinity\": " + jterms(p.required_pod_affinity) + ", \"anti\": " +
         jterms(p.required_pod_anti_affinity) + "}";
}
template <class T>
static std::string jnums(const std::vector<T>& v) {
  std::string o = "[";
  for (size_t k = 0; k < v.size(); ++k) o += (k ? ", " : "") + std::to_string((long long)v[k]);
  return o + "]";
}

struct Gen {
  std::mt19937 r;
  explicit Gen(uint32_t seed) : r(seed) {}
  uint32_t below(uint32_t n) { return r() % n; }
  bool chance(uint32_t pct) { return below(100) < pct; }
};
const char* NS[] = {"a", "b"};
const char* APPS[] = {"web", "db", "cache"};
const char* HOST = "kubernetes.io/hostname";
const char* ZONE = "topology.kubernetes.io/zone";
const char* RACK = "rack";

static PodAffinityTerm random_term(Gen& g) {
  PodAffinityTerm t;
  const uint32_t r = g.below(20);
  t.has_selector = r != 0;                       // 1 in 20 nil
  if (r == 1) {                                  // 1 in 20 invalid: Exists with a value
    t.selector.match_expressions.push_back(LabelSelectorRequirement{"tier", "Exists", {"x"}});
  } else if (r >= 3) {                           // 1 in 20 empty
    t.selector.match_labels["app"] = APPS[g.below(3)];
    if (g.chance(30)) t.selector.match_labels["tier"] = g.chance(50) ? "x" : "y";
  }
  if (g.chance(25)) t.namespaces.push_back(NS[g.below(2)]);
  const uint32_t kk = g.below(20);
  t.topology_key = kk == 0 ? "" : kk < 7 ? HOST : kk < 16 ? ZONE : RACK;
  return t;
}
static Pod random_pod(Gen& g, const std::string& name, bool bound) {
  Pod p;
  p.ns = NS[g.below(2)];
  p.name = name;
  p.uid = "uid-" + name;
  p.labels["app"] = APPS[g.below(3)];
  if (g.chance(50)) p.labels["tier"] = g.chance(50) ? "x" : "y";
  p.terminating = bound && g.chance(10);
  Container c;
  c.requests = {{"cpu", "100m"}, {"memory", "128Mi"}};
  p.containers.push_back(c);
  if (g.chance(35)) return p;
  if (!bound && g.chance(50)) {
    const uint32_t n = 1 + g.below(2);
    for (uint32_t k = 0; k < n; ++k) p.required_pod_affinity.push_back(random_term(g));
    if (g.chance(30)) {   // a self-affine set: the pod matches it itself
      PodAffinityTerm t;
      t.has_selector = true;
      t.selector.match_labels["app"] = p.labels["app"];
      t.topology_key = ZONE;
      p.required_pod_affinity.assign(1, t);
    }
  }
  if (bound || g.chance(60)) {
    const uint32_t n = 1 + g.below(2);
    for (uint32_t k = 0; k < n; ++k) p.required_pod_anti_affinity.push_back(random_term(g));
  }
  return p;
}

int main(int argc, char** argv) {
  const bool gpu = argc > 1 && !strcmp(argv[1], "gpu");
  const size_t N = 10, P = 24;
  using Choice = BatchSchedulingPlugin::ReplayNodeChoice;
  printf("{\"scenarios\": [");
  for (int sc = 0; sc < 3; ++sc) {
    Gen g(4242 + sc);
    std::vector<Node> nodes(N);
    std::vector<NodeInfo> infos(N);
    std::vector<std::vector<Pod>> bound(N);
    for (size_t i = 0; i < N; ++i) {
      nodes[i].name = "node-" + std::to_string(i);
      nodes[i].labels[HOST] = nodes[i].name;
      if (!g.chance(20)) nodes[i].labels[ZONE] = "zone-" + std::to_string(g.below(3));
      if (!g.chance(20)) nodes[i].labels[RACK] = "rack-" + std::to_string(i / 3);
      nodes[i].allocatable = {{"cpu", "64"}, {"memory", "256Gi"}, {"pods", "110"}};
      const uint32_t nb = g.below(3);
      for (uint32_t k = 0; k < nb; ++k)
        bound[i].push_back(random_pod(g, "b" + std::to_string(i) + "-" + std::to_string(k), true));
    }
    std::vector<Pod> pods;
    for (size_t p = 0; p < P; ++p) {
      pods.push_back(random_pod(g, "p" + std::to_string(p), false));
      pods.back().queue_ts_ns = (int64_t)p;
    }
    for (size_t i = 0; i < N; ++i) {
      infos[i].node = i == N - 1 ? nullptr : &nodes[i];   // the last NodeInfo has no Node: its pods count nowhere
      for (const Pod& b : bound[i]) infos[i].pods.push_back(&b);
      infos[i].num_pods = (int32_t)bound[i].size();
      infos[i].requested = {{"cpu", std::to_string(bound[i].size())}, {"memory", std::to_string(bound[i].size()) + "Gi"}};
    }
    std::vector<const NodeInfo*> snap;
    for (auto& ni : infos) snap.push_back(&ni);
    std::vector<const Pod*> pend;
    for (auto& p : pods) pend.push_back(&p);

    printf("%s{\"nodes\": [", sc ? ", " : "");
    for (size_t i = 0; i < N; ++i) {
      printf("%s{\"name\": %s, \"has_node\": %s, \"labels\": %s, \"pods\": [", i ? ", " : "", q(nodes[i].name).c_str(),
             infos[i].node ? "true" : "false", jmap(nodes[i].labels).c_str());
      for (size_t k = 0; k < bound[i].size(); ++k) printf("%s%s", k ? ", " : "", jpod(bound[i][k]).c_str());
      printf("]}");
    }
    printf("], \"pods\": [");
    for (size_t p = 0; p < P; ++p) printf("%s%s", p ? ", " : "", jpod(pods[p]).c_str());
    printf("]");
    // the filter's columns without and with the placed side
    PackedInterPodFilter plain, pk;
    Status st = BatchSchedulingPlugin::PackInterPodFilter(snap, pend, &plain);
    if (st.ok()) st = BatchSchedulingPlugin::PackInterPodFilter(snap, pend, &pk, true);
    if (!st.ok()) { fprintf(stderr, "%s\n", st.message.c_str()); return 1; }
    auto print_packed = [&](const char* name, const PackedInterPodFilter& k) {
      const PackedInterPodAffinity::Classes& bc = k.bound_classes;
      const PackedInterPodAffinity::Classes& qc = k.placed_classes;
      printf(", \"%s\": {\"keys\": %s, \"n_values\": %s, \"topo\": %s, \"term_key\": %s, \"bound_node\": %s, "
             "\"bound_class\": %s, \"bound_classes\": [%s, %s, %s, %s], \"pod_class\": %s, "
             "\"pod_classes\": [%s, %s, %s, %s], \"placed_class\": %s, \"placed_classes\": [%s, %s, %s, %s]}",
             name, jstrs(k.keys).c_str(), jnums(k.n_values).c_str(), jnums(k.topo).c_str(), jnums(k.term_key).c_str(),
             jnums(k.bound_node).c_str(), jnums(k.bound_class).c_str(), jnums(bc.offset).c_str(), jnums(bc.term).c_str(),
             jnums(bc.own).c_str(), jnums(bc.match).c_str(), jnums(k.pod_class).c_str(), jnums(k.pod_offset).c_str(),
             jnums(k.pod_term).c_str(), jnums(k.pod_role).c_str(), jnums(k.self_match).c_str(),
             jnums(k.placed_class).c_str(), jnums(qc.offset).c_str(), jnums(qc.term).c_str(), jnums(qc.own).c_str(),
             jnums(qc.match).c_str());
    };
    print_packed("plain", plain);
    print_packed("packed", pk);

    if (gpu) {
      BatchSchedulingPlugin plg(0, 0, BS_OUT_FIT_BITMAP, 0, 1);
      plg.SetInterPodAffinityFilter(true);
      Status rs = plg.BeginRound(snap, pend, 1000000000ll);
      if (!rs.ok()) { fprintf(stderr, "round failed: %s\n", rs.message.c_str()); return 1; }
      std::vector<BatchSchedulingPlugin::ReplayDecision> dec;
      const Status off = plg.ReplayQueue(&dec);
      const bool refused = !off.ok() && off.message.find("MatchInterPodAffinity") != std::string::npos;
      plg.SetInterPodAffinityFilterInWalks(true);
      rs = plg.BeginRound(snap, pend, 2000000000ll);
      if (!rs.ok()) { fprintf(stderr, "round failed: %s\n", rs.message.c_str()); return 1; }
      auto walk = [&](Choice c) {
        std::vector<BatchSchedulingPlugin::ReplayDecision> d;
        const Status s = plg.ReplayQueue(&d, c);
        if (!s.ok()) { fprintf(stderr, "replay failed: %s\n", s.message.c_str()); exit(1); }
        std::vector<int32_t> v;
        for (const auto& x : d) v.push_back(x.node);
        return v;
      };
      const std::vector<int32_t> first = walk(Choice::kFirstFit), prio = walk(Choice::kPriority);
      // UpdateNodes packs and uploads the placed side again: the walk is unchanged
      std::vector<std::pair<uint32_t, const NodeInfo*>> changed{{0u, &infos[0]}};
      const Status us = plg.UpdateNodes(changed);
      if (!us.ok()) { fprintf(stderr, "UpdateNodes failed: %s\n", us.message.c_str()); return 1; }
      const std::vector<int32_t> after_update = walk(Choice::kFirstFit);
      printf(", \"refused_without_opt_in\": %s, \"queue\": %s, \"first_fit\": %s, \"priority\": %s, "
             "\"first_fit_after_update_nodes\": %s",
             refused ? "true" : "false", jnums(plg.queue_order()).c_str(), jnums(first).c_str(), jnums(prio).c_str(),
             jnums(after_update).c_str());
    }
    printf("}");
  }
  printf("]}\n");
  return 0;
}
