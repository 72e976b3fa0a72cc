// plugin_spread_priority_test.cpp — BatchSchedulingPlugin::PackSpread and SetSelectorSpreadWeight, printed as JSON for
// tests/test_plugin_spread_priority.py (CPU) and tests/test_gpu_spread_priority.py (GPU).  One fixed round of six nodes
// (zone keys with region and zone, zone only, region only and none; bound pods in two namespaces, terminating and
// unlabelled ones) and nine pending pods, with Services (nil, empty and non-empty selectors), ReplicationControllers
// (an empty selector), ReplicaSets and StatefulSets (every operator, invalid requirements, nil and empty selectors).
// The program prints the objects themselves, so that the test evaluates them independently, and what PackSpread made
// of them; also whether 64 and 65 zones pack.  With the argument "gpu" it also runs the round on the device with
// SetSelectorSpreadWeight(1) and prints PriorityNodes next to the lists of an engine called directly with the packed
// tables, and whether ReplayQueue(kPriority) refuses the weight.
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../batch-scheduler_b200/csrc/plugin.hpp"

using namespace bsched;

static std::string q(const std::string& s) {
  std::string o = "\"";
  for (char c : s) {
    if (c == '\0') o += "\\u0000";
    else if (c == '"' || c == '\\') { o += '\\'; o += c; }
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
static std::string jls(bool has, const LabelSelector& ls) {
  if (!has) return "null";
  std::string o = "{\"match_labels\": " + jmap(ls.match_labels) + ", \"match_expressions\": [";
  for (size_t k = 0; k < ls.match_expressions.size(); ++k) {
    const auto& r = ls.match_expressions[k];
    o += (k ? ", " : "") + std::string("[") + q(r.key) + ", " + q(r.op) + ", [";
    for (size_t v = 0; v < r.values.size(); ++v) o += (v ? ", " : "") + q(r.values[v]);
    o += "]]";
  }
  return o + "]}";
}
static std::string jpod(const Pod& p) {
  return "{\"ns\": " + q(p.ns) + ", \"labels\": " + jmap(p.labels) + ", \"terminating\": " +
         (p.terminating ? "true" : "false") + "}";
}

static int packs_zones(size_t n_zones) {
  std::vector<Node> nodes(n_zones);
  std::vector<NodeInfo> infos(n_zones);
  std::vector<const NodeInfo*> snap;
  for (size_t i = 0; i < n_zones; ++i) {
    nodes[i].name = "n" + std::to_string(i);
    nodes[i].labels["failure-domain.beta.kubernetes.io/zone"] = "z" + std::to_string(i);
    infos[i].node = &nodes[i];
    snap.push_back(&infos[i]);
  }
  PackedSpread ps;
  return BatchSchedulingPlugin::PackSpread(snap, {}, SpreadSelectors{}, &ps).ok() ? (int)ps.zones.size() : -1;
}

static Pod mkpod(const std::string& ns, const std::string& name, std::map<std::string, std::string> labels,
                 bool terminating = false) {
  Pod p;
  p.ns = ns; p.name = name; p.uid = "uid-" + name;
  p.labels = std::move(labels);
  p.terminating = terminating;
  Container c;
  c.requests = {{"cpu", "1"}, {"memory", "1Gi"}};
  p.containers.push_back(c);
  return p;
}

int main(int argc, char** argv) {
  const bool gpu = argc > 1 && !strcmp(argv[1], "gpu");
  const std::string R = "failure-domain.beta.kubernetes.io/region", Z = "failure-domain.beta.kubernetes.io/zone";
  const size_t N = 6;
  std::vector<Node> nodes(N);
  std::vector<NodeInfo> infos(N);
  nodes[0].labels = {{R, "r1"}, {Z, "a"}};
  nodes[1].labels = {{R, "r1"}, {Z, "b"}};
  nodes[2].labels = {{Z, "a"}};            // zone only: another key than r1's zone a
  nodes[3].labels = {{R, "r2"}};           // region only
  nodes[4].labels = {{"rack", "7"}};       // no zone key
  nodes[5].labels = {{R, "r1"}, {Z, "a"}, {"gpu", "h100"}};
  // the pods already bound to each node (NodeInfo.Pods())
  std::vector<std::vector<Pod>> bound(N);
  bound[0] = {mkpod("default", "b0", {{"app", "web"}, {"tier", "fe"}}), mkpod("other", "b1", {{"app", "web"}}),
              mkpod("default", "b2", {{"app", "batch"}, {"role", "worker"}})};
  bound[1] = {mkpod("default", "b3", {{"app", "web"}, {"tier", "fe"}}),
              mkpod("default", "b4", {{"app", "web"}, {"tier", "fe"}}, true),   // terminating
              mkpod("default", "b5", {{"app", "batch"}, {"role", "worker"}})};
  bound[2] = {mkpod("default", "b6", {{"app", "db"}}), mkpod("default", "b7", {{"app", "batch"}, {"role", "worker"}}),
              mkpod("other", "b8", {})};
  bound[3] = {mkpod("default", "b9", {{"app", "db"}}), mkpod("default", "b10", {{"app", "web"}, {"tier", "be"}}),
              mkpod("default", "b11", {{"app", "db"}, {"tier", "x"}})};
  bound[4] = {mkpod("default", "b12", {}), mkpod("other", "b13", {{"app", "web"}}),
              mkpod("other", "b14", {{"app", "web"}}, true)};
  bound[5] = {mkpod("default", "b15", {{"app", "web"}, {"tier", "fe"}}),
              mkpod("default", "b16", {{"app", "web"}, {"tier", "fe"}}), mkpod("default", "b17", {{"app", "web"}})};
  for (size_t i = 0; i < N; ++i) {
    nodes[i].name = "node-" + std::to_string(i);
    nodes[i].allocatable = {{"cpu", "16"}, {"memory", "64Gi"}, {"pods", "110"}};
    infos[i].node = &nodes[i];
    for (const Pod& b : bound[i]) infos[i].pods.push_back(&b);
    infos[i].num_pods = (int32_t)bound[i].size();
    infos[i].requested = {{"cpu", std::to_string(bound[i].size())}, {"memory", std::to_string(bound[i].size()) + "Gi"}};
  }
  SpreadSelectors sel;
  auto svc = [](const char* ns, const char* name, bool has, std::map<std::string, std::string> s) {
    Service v; v.ns = ns; v.name = name; v.has_selector = has; v.selector = std::move(s); return v;
  };
  sel.services = {svc("default", "svc-web", true, {{"app", "web"}}), svc("default", "svc-nil", false, {}),
                  svc("other", "svc-all", true, {}), svc("default", "svc-batch", true, {{"app", "batch"}})};
  auto rc = [](const char* ns, const char* name, bool has, std::map<std::string, std::string> s) {
    ReplicationController v; v.ns = ns; v.name = name; v.has_selector = has; v.selector = std::move(s); return v;
  };
  sel.controllers = {rc("default", "rc-empty", true, {}), rc("default", "rc-db", true, {{"app", "db"}}),
                     rc("default", "rc-nil", false, {})};
  auto ls = [](std::map<std::string, std::string> ml, std::vector<LabelSelectorRequirement> me) {
    LabelSelector s; s.match_labels = std::move(ml); s.match_expressions = std::move(me); return s;
  };
  auto rs = [](const char* ns, const char* name, bool has, LabelSelector s) {
    ReplicaSet v; v.ns = ns; v.name = name; v.has_selector = has; v.selector = std::move(s); return v;
  };
  auto ss = [](const char* ns, const char* name, bool has, LabelSelector s) {
    StatefulSet v; v.ns = ns; v.name = name; v.has_selector = has; v.selector = std::move(s); return v;
  };
  sel.replica_sets = {rs("default", "rs-fe", true, ls({{"app", "web"}}, {{"tier", "In", {"fe", "be"}}})),
                      rs("default", "rs-notin", true, ls({}, {{"app", "NotIn", {"db", "web"}}, {"role", "Exists", {}}})),
                      rs("default", "rs-bad-in", true, ls({}, {{"app", "In", {}}})),
                      rs("default", "rs-bad-exists", true, ls({}, {{"app", "Exists", {"web"}}})),
                      rs("default", "rs-bad-op", true, ls({}, {{"app", "Gt", {"1"}}})),
                      rs("default", "rs-empty", true, ls({}, {})), rs("default", "rs-nil", false, ls({}, {}))};
  sel.stateful_sets = {ss("default", "ss-db", true, ls({}, {{"tier", "DoesNotExist", {}}, {"app", "In", {"db"}}})),
                       ss("other", "ss-web", true, ls({{"app", "web"}}, {})),
                       ss("default", "ss-bad-notin", true, ls({}, {{"app", "NotIn", {}}})),
                       ss("default", "ss-empty", true, ls({}, {}))};
  std::vector<Pod> pods = {mkpod("default", "p0", {{"app", "web"}, {"tier", "fe"}}),
                           mkpod("default", "p1", {{"app", "web"}}),
                           mkpod("default", "p2", {{"app", "db"}}),
                           mkpod("default", "p3", {}),
                           mkpod("other", "p4", {}),
                           mkpod("other", "p5", {{"app", "web"}}),
                           mkpod("default", "p6", {{"app", "batch"}, {"role", "worker"}}),
                           mkpod("default", "p7", {{"tier", "fe"}, {"app", "web"}}),
                           mkpod("default", "p8", {{"app", "cache"}})};
  const size_t P = pods.size();
  for (size_t p = 0; p < P; ++p) pods[p].queue_ts_ns = (int64_t)p;
  std::vector<const NodeInfo*> snap;
  for (auto& ni : infos) snap.push_back(&ni);
  std::vector<const Pod*> pend;
  for (auto& p : pods) pend.push_back(&p);

  PackedSpread ps;
  const Status st = BatchSchedulingPlugin::PackSpread(snap, pend, sel, &ps);
  if (!st.ok()) { fprintf(stderr, "%s\n", st.message.c_str()); return 1; }

  printf("{\"nodes\": [");
  for (size_t i = 0; i < N; ++i) {
    printf("%s{\"labels\": %s, \"pods\": [", i ? ", " : "", jmap(nodes[i].labels).c_str());
    for (size_t k = 0; k < bound[i].size(); ++k) printf("%s%s", k ? ", " : "", jpod(bound[i][k]).c_str());
    printf("]}");
  }
  printf("], \"pods\": [");
  for (size_t p = 0; p < P; ++p) printf("%s%s", p ? ", " : "", jpod(pods[p]).c_str());
  printf("], \"services\": [");
  for (size_t k = 0; k < sel.services.size(); ++k)
    printf("%s[%s, %s]", k ? ", " : "", q(sel.services[k].ns).c_str(),
           sel.services[k].has_selector ? jmap(sel.services[k].selector).c_str() : "null");
  printf("], \"controllers\": [");
  for (size_t k = 0; k < sel.controllers.size(); ++k)
    printf("%s[%s, %s]", k ? ", " : "", q(sel.controllers[k].ns).c_str(),
           sel.controllers[k].has_selector ? jmap(sel.controllers[k].selector).c_str() : "null");
  printf("], \"replica_sets\": [");
  for (size_t k = 0; k < sel.replica_sets.size(); ++k)
    printf("%s[%s, %s]", k ? ", " : "", q(sel.replica_sets[k].ns).c_str(),
           jls(sel.replica_sets[k].has_selector, sel.replica_sets[k].selector).c_str());
  printf("], \"stateful_sets\": [");
  for (size_t k = 0; k < sel.stateful_sets.size(); ++k)
    printf("%s[%s, %s]", k ? ", " : "", q(sel.stateful_sets[k].ns).c_str(),
           jls(sel.stateful_sets[k].has_selector, sel.stateful_sets[k].selector).c_str());
  printf("], \"zones\": [");
  for (size_t z = 0; z < ps.zones.size(); ++z) printf("%s%s", z ? ", " : "", q(ps.zones[z]).c_str());
  printf("], \"zone\": [");
  for (size_t i = 0; i < N; ++i) printf("%s%u", i ? ", " : "", (unsigned)ps.zone[i]);
  printf("], \"spread_class\": [");
  for (size_t p = 0; p < P; ++p) printf("%s%u", p ? ", " : "", ps.spread_class[p]);
  printf("], \"counts\": [");
  for (size_t k = 0; k < ps.counts.size(); ++k) printf("%s%d", k ? ", " : "", ps.counts[k]);
  printf("], \"packs_64\": %d, \"packs_65\": %d", packs_zones(64), packs_zones(65));

  if (gpu) {
    const uint32_t K = 6;
    BatchSchedulingPlugin plg(0, 0, BS_OUT_FIT_BITMAP, 0, K);
    plg.SetSpreadSelectors(sel);
    plg.SetSelectorSpreadWeight(1);
    const Status rs0 = plg.BeginRound(snap, pend, 1000000000ll);
    if (!rs0.ok()) { fprintf(stderr, "round failed: %s\n", rs0.message.c_str()); return 1; }
    std::vector<BatchSchedulingPlugin::ReplayDecision> dec;
    const bool refused = !plg.ReplayQueue(&dec, BatchSchedulingPlugin::ReplayNodeChoice::kPriority).ok();
    // the same round on an engine called directly with the packed tables
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
    if ((rc0 = bs_upload_nodes(e, &nt)) || (rc0 = bs_upload_groups(e, &gt)) || (rc0 = bs_upload_pods(e, &pt)) ||
        (rc0 = bs_upload_node_nonzero(e, N, node_nz.data())) || (rc0 = bs_upload_pod_nonzero(e, P, pod_nz.data())) ||
        (rc0 = bs_upload_node_spread(e, N, (uint32_t)ps.zones.size(), ps.zone.data(), ps.n_classes(),
                                     ps.counts.data())) ||
        (rc0 = bs_upload_pod_spread(e, P, ps.spread_class.data())) || (rc0 = bs_set_spread_weight(e, 1))) {
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
      for (auto& kv : plg.PriorityNodes(pods[p].uid)) printf("%s[%s, %lld]", k++ ? ", " : "", q(kv.first).c_str(), (long long)kv.second);
      printf("]");
    }
    printf("], \"engine\": [");
    for (size_t p = 0; p < P; ++p) {
      printf("%s[", p ? ", " : "");
      for (uint32_t k = 0; k < K && en[p * K + k] >= 0; ++k)
        printf("%s[%s, %lld]", k ? ", " : "", q(nodes[en[p * K + k]].name).c_str(), (long long)es[p * K + k]);
      printf("]");
    }
    printf("]");
  }
  printf("}\n");
  return 0;
}
