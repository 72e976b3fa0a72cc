// plugin_reasons_test.cpp — BatchSchedulingPlugin created with BS_OUT_REASONS: after BeginRound and after an
// UpdateRound, prints for every pending pod its feasible count, ReasonCounts(uid) and FitError(uid), as JSON for
// tests/test_gpu_fit_reasons.py.
//   reasons   (GPU)
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../batch-scheduler_b200/csrc/plugin.hpp"

using namespace bsched;

static std::string json_str(const std::string& s) {
  std::string o = "\"";
  for (char c : s) {
    if (c == '"' || c == '\\') o += '\\';
    o += c;
  }
  return o + "\"";
}

static void print_round(const BatchSchedulingPlugin& plugin, const std::vector<Pod>& pods, bool last) {
  printf("{\"lanes\": %u, \"feasible\": [", plugin.packed().lanes);
  for (size_t i = 0; i < pods.size(); ++i) printf("%s%u", i ? ", " : "", plugin.feasible_counts()[i]);
  printf("], \"counts\": [");
  for (size_t i = 0; i < pods.size(); ++i) {
    printf("%s[", i ? ", " : "");
    const auto c = plugin.ReasonCounts(pods[i].uid);
    for (size_t b = 0; b < c.size(); ++b) printf("%s%u", b ? ", " : "", c[b]);
    printf("]");
  }
  printf("], \"errors\": [");
  for (size_t i = 0; i < pods.size(); ++i) printf("%s%s", i ? ", " : "", json_str(plugin.FitError(pods[i].uid)).c_str());
  printf("], \"unknown\": [%zu, %s]}%s\n", plugin.ReasonCounts("no-such-uid").size(),
         json_str(plugin.FitError("no-such-uid")).c_str(), last ? "" : ",");
}

static int cmd_reasons() {
  // 10 nodes: 0-3 with 4 cpus and 1 of 2 GPUs free, 4-5 without GPUs, 6 unschedulable, 7 tainted, 8 without a Node
  // object, 9 with 64 cpus and the label zone=b but no GPU key
  const int N = 10;
  std::vector<Node> nodes(N);
  std::vector<NodeInfo> infos(N);
  for (int i = 0; i < N; ++i) {
    Node& n = nodes[i];
    n.name = "node-" + std::to_string(i);
    n.allocatable = {{"cpu", "4"}, {"memory", "8Gi"}, {"pods", "110"}};
    infos[i].node = &n;
    if (i < 4) {
      n.allocatable.push_back({"nvidia.com/gpu", "2"});
      infos[i].requested = {{"cpu", "0"}, {"nvidia.com/gpu", "1"}};
    }
  }
  nodes[6].unschedulable = true;
  nodes[7].taints = {{"dedicated", "infra", "NoSchedule"}};
  nodes[7].allocatable = {{"cpu", "64"}, {"memory", "64Gi"}, {"pods", "110"}};
  infos[8].node = nullptr;
  nodes[9].labels = {{"zone", "b"}};
  nodes[9].allocatable = {{"cpu", "64"}, {"memory", "64Gi"}, {"pods", "110"}};

  auto make_pod = [](int i, const char* cpu, const char* gpu) {
    Pod p;
    p.ns = "default"; p.name = "pod-" + std::to_string(i); p.uid = "uid-" + std::to_string(i);
    Container c;
    c.has_limits = true;
    c.limits = {{"cpu", cpu}};
    if (gpu) c.limits.push_back({"nvidia.com/gpu", gpu});
    p.containers = {c};
    p.queue_ts_ns = i;
    return p;
  };
  std::vector<Pod> pods;
  pods.push_back(make_pod(0, "8", "1"));       // too much cpu for nodes 0-5, no GPU on 4, 5 and 9
  pods.push_back(make_pod(1, "100", nullptr)); // only node 9 matches its selector, and it has too few cpus
  pods[1].node_selector = {{"zone", "b"}};
  pods.push_back(make_pod(2, "1", nullptr));   // fits
  BatchSchedulingPlugin plugin(0, 0, BS_OUT_FIT_BITMAP | BS_OUT_REASONS);
  std::vector<const NodeInfo*> snap(N);
  std::vector<const Pod*> pend;
  for (int i = 0; i < N; ++i) snap[i] = &infos[i];
  for (auto& p : pods) pend.push_back(&p);
  Status st = plugin.BeginRound(snap, pend, 1000000000ll);
  if (!st.ok()) { fprintf(stderr, "round failed: %s\n", st.message.c_str()); return 1; }
  printf("[\n");
  print_round(plugin, pods, false);
  // node 6 becomes schedulable with 64 cpus and 4 free GPUs: pod 0 fits there now, pod 1 loses its unschedulable node
  // to the selector bin
  nodes[6].unschedulable = false;
  nodes[6].allocatable = {{"cpu", "64"}, {"memory", "64Gi"}, {"pods", "110"}, {"nvidia.com/gpu", "4"}};
  infos[6].requested = {{"cpu", "0"}, {"nvidia.com/gpu", "0"}};
  st = plugin.UpdateRound({{6u, &infos[6]}}, {}, 2000000000ll);
  if (!st.ok()) { fprintf(stderr, "update failed: %s\n", st.message.c_str()); return 1; }
  print_round(plugin, pods, true);
  printf("]\n");
  return 0;
}

int main(int argc, char** argv) {
  if (argc >= 2 && !strcmp(argv[1], "reasons")) return cmd_reasons();
  fprintf(stderr, "usage: %s reasons\n", argv[0]);
  return 2;
}
