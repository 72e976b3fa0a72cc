// plugin_node_priority_test.cpp — BatchSchedulingPlugin::PackPreferences and SetNodePriorityWeights, printed as JSON for
// tests/test_plugin_node_priority.py (CPU) and tests/test_gpu_node_priority.py (GPU).  One fixed round of six nodes
// (labels, PreferNoSchedule taints, one NoSchedule taint) and nine pending pods (tolerations of every effect and
// operator, preferred terms with every operator, empty expressions, match_fields, weight 0 and an invalid requirement).
// The program prints the objects themselves, so that the test evaluates them independently, and what PackPreferences
// made of them; also whether 64 and 65 distinct PreferNoSchedule taints pack.  With the argument "gpu" it also runs the
// round on the device with SetNodePriorityWeights(1, 1) and prints PriorityNodes of every pod next to the lists of an
// engine called directly with the packed tables, and whether ReplayQueue(kPriority) refuses to run.
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../batch-scheduler_b200/csrc/plugin.hpp"

using namespace bsched;

static std::string q(const std::string& s) { return "\"" + s + "\""; }

static NodeSelectorRequirement req(const std::string& key, const std::string& op, std::vector<std::string> values) {
  NodeSelectorRequirement r;
  r.key = key; r.op = op; r.values = std::move(values);
  return r;
}
static PreferredSchedulingTerm term(int32_t w, std::vector<NodeSelectorRequirement> exprs,
                                    std::vector<NodeSelectorRequirement> fields = {}) {
  PreferredSchedulingTerm t;
  t.weight = w;
  t.preference.match_expressions = std::move(exprs);
  t.preference.match_fields = std::move(fields);
  return t;
}

static void print_reqs(const std::vector<NodeSelectorRequirement>& rs) {
  printf("[");
  for (size_t i = 0; i < rs.size(); ++i) {
    printf("%s[%s, %s, [", i ? ", " : "", q(rs[i].key).c_str(), q(rs[i].op).c_str());
    for (size_t k = 0; k < rs[i].values.size(); ++k) printf("%s%s", k ? ", " : "", q(rs[i].values[k]).c_str());
    printf("]]");
  }
  printf("]");
}

static int packs(size_t n_taints) {
  std::vector<Node> nodes(n_taints);
  std::vector<NodeInfo> infos(n_taints);
  std::vector<const NodeInfo*> snap;
  for (size_t i = 0; i < n_taints; ++i) {
    nodes[i].name = "n" + std::to_string(i);
    nodes[i].taints = {Taint{"k", std::to_string(i), "PreferNoSchedule"}, Taint{"k", "0", "PreferNoSchedule"}};
    infos[i].node = &nodes[i];
    snap.push_back(&infos[i]);
  }
  PackedPreferences pp;
  return BatchSchedulingPlugin::PackPreferences(snap, {}, &pp).ok() ? (int)pp.taints.size() : -1;
}

int main(int argc, char** argv) {
  const bool gpu = argc > 1 && !strcmp(argv[1], "gpu");
  const size_t N = 6, P = 9;
  std::vector<Node> nodes(N);
  std::vector<NodeInfo> infos(N);
  nodes[0].labels = {{"zone", "a"}, {"rack", "1"}, {"gen", "5"}};
  nodes[0].taints = {{"k1", "v1", "PreferNoSchedule"}};
  nodes[1].labels = {{"zone", "b"}, {"rack", "2"}, {"gen", "10"}};
  nodes[1].taints = {{"k1", "v2", "PreferNoSchedule"}, {"k2", "", "PreferNoSchedule"}};
  nodes[2].labels = {{"zone", "a"}, {"rack", "3"}};
  nodes[2].taints = {{"k3", "x", "NoSchedule"}, {"k2", "", "PreferNoSchedule"}};
  nodes[3].labels = {{"zone", "c"}, {"gen", "abc"}};
  nodes[4].taints = {{"k1", "v1", "PreferNoSchedule"}, {"k4", "z", "PreferNoSchedule"}};
  nodes[5].labels = {{"zone", "a"}, {"gen", "7"}};
  nodes[5].taints = {{"k2", "", "PreferNoSchedule"}, {"k1", "v1", "PreferNoSchedule"}, {"k5", "y", "NoExecute"}};
  for (size_t i = 0; i < N; ++i) {
    nodes[i].name = "node-" + std::to_string(i);
    nodes[i].allocatable = {{"cpu", "16"}, {"memory", "64Gi"}, {"pods", "110"}};
    infos[i].node = &nodes[i];
  }
  std::vector<Pod> pods(P);
  pods[1].tolerations = {{"k1", "Equal", "v1", ""}, {"k2", "Exists", "", "NoSchedule"}};
  pods[2].tolerations = {{"", "Exists", "", "PreferNoSchedule"}, {"k5", "Exists", "", "NoExecute"}};
  pods[3].tolerations = {{"k1", "Exists", "", "PreferNoSchedule"}, {"k4", "", "z", ""}, {"k3", "Equal", "x", ""}};
  const std::vector<PreferredSchedulingTerm> mixed = {
      term(10, {req("zone", "In", {"a"})}),
      term(5, {req("gen", "Gt", {"6"})}),
      term(0, {req("rack", "Exists", {})}),
      term(7, {}, {req("metadata.name", "In", {"node-0"})}),
      term(3, {req("zone", "In", {})}),
      term(2, {req("rack", "NotIn", {"1"}), req("gen", "DoesNotExist", {})}),
  };
  pods[4].preferred_affinity = mixed;
  pods[5].preferred_affinity = mixed;
  pods[5].tolerations = {{"k2", "Equal", "", "PreferNoSchedule"}};
  pods[6].preferred_affinity = {term(4, {req("gen", "Lt", {"7"})}), term(9, {req("zone", "Exists", {})})};
  pods[7].preferred_affinity = {term(0, {req("zone", "In", {"a"})})};
  pods[8].preferred_affinity = {term(10, {req("zone", "In", {"a"})}), term(1, {req("rack", "Gt", {"x"})})};
  pods[8].tolerations = {{"", "Exists", "", ""}};
  for (size_t p = 0; p < P; ++p) {
    pods[p].ns = "default"; pods[p].name = "pod-" + std::to_string(p); pods[p].uid = "uid-" + std::to_string(p);
    Container c;
    c.requests = {{"cpu", "1"}, {"memory", "1Gi"}};
    pods[p].containers = {c};
    pods[p].queue_ts_ns = (int64_t)p;
  }
  std::vector<const NodeInfo*> snap;
  for (auto& ni : infos) snap.push_back(&ni);
  std::vector<const Pod*> pend;
  for (auto& p : pods) pend.push_back(&p);

  PackedPreferences pp;
  const Status st = BatchSchedulingPlugin::PackPreferences(snap, pend, &pp);
  if (!st.ok()) { fprintf(stderr, "%s\n", st.message.c_str()); return 1; }

  printf("{\"nodes\": [");
  for (size_t i = 0; i < N; ++i) {
    printf("%s{\"labels\": {", i ? ", " : "");
    size_t k = 0;
    for (auto& kv : nodes[i].labels) printf("%s%s: %s", k++ ? ", " : "", q(kv.first).c_str(), q(kv.second).c_str());
    printf("}, \"taints\": [");
    for (size_t t = 0; t < nodes[i].taints.size(); ++t)
      printf("%s[%s, %s, %s]", t ? ", " : "", q(nodes[i].taints[t].key).c_str(), q(nodes[i].taints[t].value).c_str(),
             q(nodes[i].taints[t].effect).c_str());
    printf("]}");
  }
  printf("], \"pods\": [");
  for (size_t p = 0; p < P; ++p) {
    printf("%s{\"tolerations\": [", p ? ", " : "");
    for (size_t t = 0; t < pods[p].tolerations.size(); ++t) {
      const Toleration& o = pods[p].tolerations[t];
      printf("%s[%s, %s, %s, %s]", t ? ", " : "", q(o.key).c_str(), q(o.op).c_str(), q(o.value).c_str(), q(o.effect).c_str());
    }
    printf("], \"preferred\": [");
    for (size_t t = 0; t < pods[p].preferred_affinity.size(); ++t) {
      printf("%s[%d, ", t ? ", " : "", pods[p].preferred_affinity[t].weight);
      print_reqs(pods[p].preferred_affinity[t].preference.match_expressions);
      printf(", ");
      print_reqs(pods[p].preferred_affinity[t].preference.match_fields);
      printf("]");
    }
    printf("]}");
  }
  printf("], \"dict\": [");
  for (size_t b = 0; b < pp.taints.size(); ++b) printf("%s[%s, %s]", b ? ", " : "", q(pp.taints[b].key).c_str(), q(pp.taints[b].value).c_str());
  printf("], \"prefer_taints\": [");
  for (size_t i = 0; i < N; ++i) printf("%s%llu", i ? ", " : "", (unsigned long long)pp.prefer_taints[i]);
  printf("], \"prefer_tol\": [");
  for (size_t p = 0; p < P; ++p) printf("%s%llu", p ? ", " : "", (unsigned long long)pp.prefer_tol[p]);
  printf("], \"pref_class\": [");
  for (size_t p = 0; p < P; ++p) printf("%s%u", p ? ", " : "", pp.pref_class[p]);
  printf("], \"pref_weights\": [");
  for (uint32_t c = 0; c < pp.n_classes(); ++c) {
    printf("%s[", c ? ", " : "");
    for (size_t i = 0; i < N; ++i) printf("%s%d", i ? ", " : "", pp.pref_weights[c * N + i]);
    printf("]");
  }
  printf("], \"packs_64\": %d, \"packs_65\": %d", packs(64), packs(65));

  if (gpu) {
    const uint32_t K = 6;
    BatchSchedulingPlugin pl(0, 0, BS_OUT_FIT_BITMAP, 0, K);
    pl.SetNodePriorityWeights(1, 1);
    const Status rs = pl.BeginRound(snap, pend, 1000000000ll);
    if (!rs.ok()) { fprintf(stderr, "round failed: %s\n", rs.message.c_str()); return 1; }
    std::vector<BatchSchedulingPlugin::ReplayDecision> dec;
    const Status refused = pl.ReplayQueue(&dec, BatchSchedulingPlugin::ReplayNodeChoice::kPriority);
    // the same round on an engine called directly with the packed tables
    const PackedSnapshot& ps = pl.packed();
    bs_config cfg{0, ps.lanes, BS_OUT_PRIORITY, K};
    bs_engine* e = nullptr;
    int rc = bs_create(&cfg, &e);
    if (rc) { fprintf(stderr, "bs_create: %d\n", rc); return 1; }
    const bs_node_table nt = ps.node_table();
    const bs_group_table gt = ps.group_table();
    const bs_pod_table pt = ps.pod_table();
    std::vector<int64_t> node_nz, pod_nz;
    BatchSchedulingPlugin::PackNonZero(snap, pend, &node_nz, &pod_nz);
    if ((rc = bs_upload_nodes(e, &nt)) || (rc = bs_upload_groups(e, &gt)) || (rc = bs_upload_pods(e, &pt)) ||
        (rc = bs_upload_node_nonzero(e, N, node_nz.data())) || (rc = bs_upload_pod_nonzero(e, P, pod_nz.data())) ||
        (rc = bs_upload_node_preferences(e, N, pp.prefer_taints.data(), pp.n_classes(), pp.pref_weights.data())) ||
        (rc = bs_upload_pod_preferences(e, P, pp.prefer_tol.data(), pp.pref_class.data())) ||
        (rc = bs_set_node_priority_weights(e, 1, 1))) {
      fprintf(stderr, "engine setup: %d %s\n", rc, bs_last_error(e));
      return 1;
    }
    bs_results res{};
    if ((rc = bs_evaluate(e, &res))) { fprintf(stderr, "bs_evaluate: %d\n", rc); return 1; }
    std::vector<int32_t> en(P * K);
    std::vector<int64_t> es(P * K);
    if ((rc = bs_fetch_priority_rows(e, 0, P, en.data(), es.data()))) { fprintf(stderr, "fetch: %d\n", rc); return 1; }
    bs_destroy(e);
    printf(", \"replay_refused\": %d, \"plugin\": [", refused.ok() ? 0 : 1);
    for (size_t p = 0; p < P; ++p) {
      printf("%s[", p ? ", " : "");
      size_t k = 0;
      for (auto& kv : pl.PriorityNodes(pods[p].uid)) printf("%s[%s, %lld]", k++ ? ", " : "", q(kv.first).c_str(), (long long)kv.second);
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
