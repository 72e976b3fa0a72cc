// plugin_interpod_priority_test.cpp — BatchSchedulingPlugin::PackInterPodAffinity and SetInterPodAffinityWeight,
// printed as JSON for tests/test_plugin_interpod_priority.py (CPU) and tests/test_gpu_interpod_priority.py (GPU).
// Seeded rounds of twelve nodes (hostname, zone and rack keys, some nodes without the zone or rack key) with bound pods
// and pending pods in three namespaces whose required and preferred pod-affinity and preferred anti-affinity terms
// use nil and empty selectors, every operator, listed and empty namespaces and an empty topology key; one scenario
// adds a pending pod's invalid selector, one a bound pod's.  The program prints the objects, so that the test packs
// them independently, and what PackInterPodAffinity made of them at hard weights 0, 1 and 100; also whether 64 and 65
// topology keys pack, and whether SetHardPodAffinityWeight takes -1, 0, 100 and 101.  With the argument "gpu" it also
// runs a round on the device with SetInterPodAffinityWeight(1) and prints PriorityNodes next to the lists of an engine
// called directly with the packed tables, and whether ReplayQueue(kPriority) refuses the weight.
#include <cstdio>
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
static std::string jterm(const PodAffinityTerm& t) {
  std::string o = "{\"selector\": ";
  if (!t.has_selector) {
    o += "null";
  } else {
    o += "{\"match_labels\": " + jmap(t.selector.match_labels) + ", \"match_expressions\": [";
    for (size_t k = 0; k < t.selector.match_expressions.size(); ++k) {
      const auto& r = t.selector.match_expressions[k];
      o += (k ? ", " : "") + std::string("[") + q(r.key) + ", " + q(r.op) + ", " + jstrs(r.values) + "]";
    }
    o += "]}";
  }
  return o + ", \"namespaces\": " + jstrs(t.namespaces) + ", \"key\": " + q(t.topology_key) + "}";
}
static std::string jpod(const Pod& p) {
  std::string o = "{\"ns\": " + q(p.ns) + ", \"labels\": " + jmap(p.labels) + ", \"terminating\": " +
                  (p.terminating ? "true" : "false") + ", \"required\": [";
  for (size_t k = 0; k < p.required_pod_affinity.size(); ++k) o += (k ? ", " : "") + jterm(p.required_pod_affinity[k]);
  o += "], \"preferred\": [";
  for (size_t k = 0; k < p.preferred_pod_affinity.size(); ++k)
    o += (k ? ", " : "") + std::string("[") + std::to_string(p.preferred_pod_affinity[k].weight) + ", " +
         jterm(p.preferred_pod_affinity[k].term) + "]";
  o += "], \"anti\": [";
  for (size_t k = 0; k < p.preferred_pod_anti_affinity.size(); ++k)
    o += (k ? ", " : "") + std::string("[") + std::to_string(p.preferred_pod_anti_affinity[k].weight) + ", " +
         jterm(p.preferred_pod_anti_affinity[k].term) + "]";
  return o + "]}";
}
template <class T>
static std::string jnums(const std::vector<T>& v) {
  std::string o = "[";
  for (size_t k = 0; k < v.size(); ++k) o += (k ? ", " : "") + std::to_string((long long)v[k]);
  return o + "]";
}
static std::string jclasses(const PackedInterPodAffinity::Classes& c) {
  return "[" + jnums(c.offset) + ", " + jnums(c.term) + ", " + jnums(c.own) + ", " + jnums(c.match) + "]";
}

// a seeded generator over raw mt19937 draws (portable across standard libraries)
struct Gen {
  std::mt19937 r;
  explicit Gen(uint32_t seed) : r(seed) {}
  uint32_t below(uint32_t n) { return r() % n; }
  bool chance(uint32_t pct) { return below(100) < pct; }
};
const char* NS[] = {"a", "b", "c"};
const char* APPS[] = {"web", "db", "cache", "batch"};
const char* HOST = "kubernetes.io/hostname";
const char* ZONE = "failure-domain.beta.kubernetes.io/zone";
const char* RACK = "rack";

static PodAffinityTerm random_term(Gen& g) {
  PodAffinityTerm t;
  const uint32_t r = g.below(10);
  t.has_selector = r != 0;   // 1 in 10 nil
  if (r >= 2) {              // 1 in 10 empty
    if (g.chance(70)) t.selector.match_labels["app"] = APPS[g.below(4)];
    if (g.chance(40)) {
      static const char* ops[] = {"In", "NotIn", "Exists", "DoesNotExist"};
      LabelSelectorRequirement q{"tier", ops[g.below(4)], {}};
      if (q.op == "In" || q.op == "NotIn") {
        q.values.push_back(g.chance(50) ? "x" : "y");
        if (g.chance(40)) q.values.push_back("x");
      }
      t.selector.match_expressions.push_back(q);
    }
  }
  if (g.chance(40)) {
    const uint32_t k = 1 + g.below(2);
    for (uint32_t i = 0; i < k; ++i) t.namespaces.push_back(NS[g.below(3)]);
  }
  const uint32_t kk = g.below(20);
  t.topology_key = kk == 0 ? "" : kk < 6 ? HOST : kk < 15 ? ZONE : RACK;
  return t;
}
static Pod random_pod(Gen& g, const std::string& name) {
  Pod p;
  p.ns = NS[g.below(3)];
  p.name = name;
  p.uid = "uid-" + name;
  p.labels["app"] = APPS[g.below(4)];
  if (g.chance(50)) p.labels["tier"] = g.chance(50) ? "x" : "z";
  p.terminating = g.chance(10);
  Container c;
  c.requests = {{"cpu", "1"}, {"memory", "1Gi"}};
  p.containers.push_back(c);
  if (g.chance(30)) return p;
  const uint32_t n = g.below(4);
  for (uint32_t k = 0; k < n; ++k) {
    const uint32_t kind = g.below(3);
    const int32_t w = 1 + (int32_t)g.below(100);
    if (kind == 0) p.required_pod_affinity.push_back(random_term(g));
    else if (kind == 1) p.preferred_pod_affinity.push_back(WeightedPodAffinityTerm{w, random_term(g)});
    else p.preferred_pod_anti_affinity.push_back(WeightedPodAffinityTerm{w, random_term(g)});
  }
  return p;
}
static PodAffinityTerm invalid_term() {
  PodAffinityTerm t;
  t.has_selector = true;
  t.selector.match_expressions.push_back(LabelSelectorRequirement{"tier", "Exists", {"x"}});
  t.topology_key = HOST;
  return t;
}

static int packs_keys(size_t n_keys) {
  Node node;
  node.name = "n0";
  NodeInfo ni;
  ni.node = &node;
  std::vector<const NodeInfo*> snap{&ni};
  Pod p;
  p.ns = "a";
  for (size_t k = 0; k < n_keys; ++k) {
    PodAffinityTerm t;
    t.has_selector = true;
    t.topology_key = "key-" + std::to_string(k);
    p.preferred_pod_affinity.push_back(WeightedPodAffinityTerm{1, t});
  }
  PackedInterPodAffinity pk;
  return BatchSchedulingPlugin::PackInterPodAffinity(snap, {&p}, 1, &pk).ok() ? (int)pk.keys.size() : -1;
}

int main(int argc, char** argv) {
  const bool gpu = argc > 1 && !strcmp(argv[1], "gpu");
  const size_t N = 12, P = 15;
  printf("{\"scenarios\": [");
  for (int sc = 0; sc < 3; ++sc) {
    Gen g(1234 + sc);
    std::vector<Node> nodes(N);
    std::vector<NodeInfo> infos(N);
    std::vector<std::vector<Pod>> bound(N);
    for (size_t i = 0; i < N; ++i) {
      nodes[i].name = "node-" + std::to_string(i);
      nodes[i].labels[HOST] = nodes[i].name;
      if (!g.chance(15)) nodes[i].labels[ZONE] = "zone-" + std::to_string(g.below(3));
      if (!g.chance(15)) nodes[i].labels[RACK] = "rack-" + std::to_string(i / 4);
      nodes[i].allocatable = {{"cpu", "16"}, {"memory", "64Gi"}, {"pods", "110"}};
      const uint32_t nb = g.below(5);
      for (uint32_t k = 0; k < nb; ++k) bound[i].push_back(random_pod(g, "b" + std::to_string(i) + "-" + std::to_string(k)));
    }
    std::vector<Pod> pods;
    for (size_t p = 0; p < P; ++p) {
      pods.push_back(random_pod(g, "p" + std::to_string(p)));
      pods.back().queue_ts_ns = (int64_t)p;
    }
    if (sc >= 1) pods[4].preferred_pod_affinity.push_back(WeightedPodAffinityTerm{5, invalid_term()});
    if (sc == 2) bound[3].push_back(Pod(pods[0])), bound[3].back().preferred_pod_anti_affinity.push_back(
                                                       WeightedPodAffinityTerm{5, invalid_term()});
    for (size_t i = 0; i < N; ++i) {
      infos[i].node = &nodes[i];
      for (const Pod& b : bound[i]) infos[i].pods.push_back(&b);
      infos[i].num_pods = (int32_t)bound[i].size();
      infos[i].requested = {{"cpu", std::to_string(bound[i].size())},
                            {"memory", std::to_string(bound[i].size()) + "Gi"}};
    }
    std::vector<const NodeInfo*> snap;
    for (auto& ni : infos) snap.push_back(&ni);
    std::vector<const Pod*> pend;
    for (auto& p : pods) pend.push_back(&p);

    printf("%s{\"nodes\": [", sc ? ", " : "");
    for (size_t i = 0; i < N; ++i) {
      printf("%s{\"labels\": %s, \"pods\": [", i ? ", " : "", jmap(nodes[i].labels).c_str());
      for (size_t k = 0; k < bound[i].size(); ++k) printf("%s%s", k ? ", " : "", jpod(bound[i][k]).c_str());
      printf("]}");
    }
    printf("], \"pods\": [");
    for (size_t p = 0; p < P; ++p) printf("%s%s", p ? ", " : "", jpod(pods[p]).c_str());
    printf("], \"packed\": {");
    for (int hard : {0, 1, 100}) {
      PackedInterPodAffinity pk;
      const Status st = BatchSchedulingPlugin::PackInterPodAffinity(snap, pend, hard, &pk);
      if (!st.ok()) { fprintf(stderr, "%s\n", st.message.c_str()); return 1; }
      printf("%s\"%d\": {\"keys\": %s, \"values\": [", hard ? ", " : "", hard, jstrs(pk.keys).c_str());
      for (size_t k = 0; k < pk.values.size(); ++k) printf("%s%s", k ? ", " : "", jstrs(pk.values[k]).c_str());
      printf("], \"n_values\": %s, \"topo\": %s, \"term_key\": %s, \"bound_node\": %s, \"bound_class\": %s, "
             "\"bound_classes\": %s, \"pod_class\": %s, \"pod_classes\": %s}",
             jnums(pk.n_values).c_str(), jnums(pk.topo).c_str(), jnums(pk.term_key).c_str(),
             jnums(pk.bound_node).c_str(), jnums(pk.bound_class).c_str(), jclasses(pk.bound_classes).c_str(),
             jnums(pk.pod_class).c_str(), jclasses(pk.pod_classes).c_str());
    }
    printf("}");

    if (gpu && sc == 0) {
      const uint32_t K = 6;
      BatchSchedulingPlugin plg(0, 0, BS_OUT_FIT_BITMAP, 0, K);
      plg.SetInterPodAffinityWeight(1);
      const Status rs0 = plg.BeginRound(snap, pend, 1000000000ll);
      if (!rs0.ok()) { fprintf(stderr, "round failed: %s\n", rs0.message.c_str()); return 1; }
      std::vector<BatchSchedulingPlugin::ReplayDecision> dec;
      const bool refused = !plg.ReplayQueue(&dec, BatchSchedulingPlugin::ReplayNodeChoice::kPriority).ok();
      // the same round on an engine called directly with the packed tables
      PackedInterPodAffinity ip;
      if (!BatchSchedulingPlugin::PackInterPodAffinity(snap, pend, 1, &ip).ok()) return 1;
      const PackedSnapshot& pk = plg.packed();
      bs_config cfg{0, pk.lanes, BS_OUT_PRIORITY, K};
      bs_engine* e = nullptr;
      int rc0 = bs_create(&cfg, &e);
      if (rc0) { fprintf(stderr, "bs_create: %d\n", rc0); return 1; }
      const bs_node_table nt = pk.node_table();
      const bs_group_table gt = pk.group_table();
      const bs_pod_table pt = pk.pod_table();
      std::vector<int64_t> node_nz, pod_nz;
      BatchSchedulingPlugin::PackNonZero(snap, pend, &node_nz, &pod_nz);
      auto cl = [](const PackedInterPodAffinity::Classes& c) {
        return bs_interpod_classes{c.n_classes(), c.offset.data(), c.term.data(), c.own.data(), c.match.data()};
      };
      const bs_interpod_nodes in{(uint32_t)N, (uint32_t)ip.keys.size(), ip.n_values.data(), ip.topo.data(),
                                 (uint32_t)ip.term_key.size(), ip.term_key.data(), (uint32_t)ip.bound_node.size(),
                                 ip.bound_node.data(), ip.bound_class.data(), cl(ip.bound_classes)};
      const bs_interpod_pods ipp{(uint32_t)P, ip.pod_class.data(), cl(ip.pod_classes)};
      if ((rc0 = bs_upload_nodes(e, &nt)) || (rc0 = bs_upload_groups(e, &gt)) || (rc0 = bs_upload_pods(e, &pt)) ||
          (rc0 = bs_upload_node_nonzero(e, N, node_nz.data())) || (rc0 = bs_upload_pod_nonzero(e, P, pod_nz.data())) ||
          (rc0 = bs_upload_node_interpod(e, &in)) || (rc0 = bs_upload_pod_interpod(e, &ipp)) ||
          (rc0 = bs_set_interpod_weight(e, 1))) {
        fprintf(stderr, "engine setup: %d %s\n", rc0, bs_last_error(e));
        return 1;
      }
      bs_results res{};
      if ((rc0 = bs_evaluate(e, &res))) { fprintf(stderr, "bs_evaluate: %d\n", rc0); return 1; }
      std::vector<int32_t> en(P * K);
      std::vector<int64_t> es(P * K);
      if ((rc0 = bs_fetch_priority_rows(e, 0, P, en.data(), es.data()))) { fprintf(stderr, "fetch: %d\n", rc0); return 1; }
      bs_destroy(e);
      printf(", \"replay_refused\": %s, \"plugin\": [", refused ? "true" : "false");
      for (size_t p = 0; p < P; ++p) {
        printf("%s[", p ? ", " : "");
        size_t k = 0;
        for (auto& kv : plg.PriorityNodes(pods[p].uid))
          printf("%s[%s, %lld]", k++ ? ", " : "", q(kv.first).c_str(), (long long)kv.second);
        printf("]");
      }
      printf("], \"engine\": [");
      for (size_t p = 0; p < P; ++p) {
        printf("%s[", p ? ", " : "");
        for (uint32_t k = 0; k < K && en[p * K + k] >= 0; ++k)
          printf("%s[%s, %lld]", k ? ", " : "", q(nodes[en[p * K + k]].name).c_str(), (long long)es[p * K + k]);
        printf("]");
      }
      printf("], \"n_nodes\": %zu", N);
    }
    printf("}");
  }
  BatchSchedulingPlugin probe(0, 0, BS_OUT_FIT_BITMAP, 0, 0);
  printf("], \"packs_64\": %d, \"packs_65\": %d, \"hard_weight_ok\": [", packs_keys(64), packs_keys(65));
  int k = 0;
  for (int w : {-1, 0, 100, 101}) printf("%s%s", k++ ? ", " : "", probe.SetHardPodAffinityWeight(w).ok() ? "true" : "false");
  printf("]}\n");
  return 0;
}
