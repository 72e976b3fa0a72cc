// plugin_priority_test.cpp — the resource priorities through BatchSchedulingPlugin, printed as JSON for
// tests/test_priority_oracle.py (pack, no GPU) and tests/test_gpu_priority.py (round, GPU).
//   pack    PackNonZero's columns for pods with absent, explicit-zero and set requests, and NodeInfos listing them
//   round   a three-node cluster where the LeastAllocated pick, the MostAllocated pick and the min-residual
//           best_node are three different nodes: PriorityNodes after BeginRound and after an UpdateRound
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../batch-scheduler_b200/csrc/plugin.hpp"

using namespace bsched;

static void print_list(const std::vector<int64_t>& v, bool last) {
  printf("[");
  for (size_t i = 0; i < v.size(); ++i) printf("%s%lld", i ? ", " : "", (long long)v[i]);
  printf("]%s", last ? "" : ", ");
}

static int cmd_pack() {
  std::vector<Pod> pods(7);
  auto req = [](ResourceList r) { Container c; c.requests = std::move(r); return c; };
  pods[1].containers = {req({})};
  pods[2].containers = {req({{"cpu", "0"}, {"memory", "0"}})};
  pods[3].containers = {req({{"cpu", "1500m"}, {"memory", "3Gi"}})};
  pods[4].containers = {req({{"cpu", "250m"}})};
  pods[5].containers = {req({{"cpu", "250m"}, {"memory", "1Gi"}}), req({})};
  Container lim;
  lim.has_limits = true;
  lim.limits = {{"cpu", "2"}, {"memory", "8Gi"}};
  pods[6].containers = {lim};   // Requests, not Limits, count: both keys absent
  std::vector<const Pod*> pend;
  for (auto& p : pods) pend.push_back(&p);
  Node n;
  n.name = "n";
  std::vector<NodeInfo> infos(3);
  for (auto& ni : infos) ni.node = &n;
  infos[1].pods = {&pods[1], &pods[3]};
  infos[2].pods = {&pods[4], &pods[5]};
  std::vector<const NodeInfo*> snap = {&infos[0], &infos[1], &infos[2], nullptr};
  std::vector<int64_t> node_nz, pod_nz;
  Status st = BatchSchedulingPlugin::PackNonZero(snap, pend, &node_nz, &pod_nz);
  if (!st.ok()) { fprintf(stderr, "%s\n", st.message.c_str()); return 1; }
  const size_t P = pods.size(), N = snap.size();
  printf("{\"pod_cpu\": ");
  print_list(std::vector<int64_t>(pod_nz.begin(), pod_nz.begin() + P), false);
  printf("\"pod_mem\": ");
  print_list(std::vector<int64_t>(pod_nz.begin() + P, pod_nz.end()), false);
  printf("\"node_cpu\": ");
  print_list(std::vector<int64_t>(node_nz.begin(), node_nz.begin() + N), false);
  printf("\"node_mem\": ");
  print_list(std::vector<int64_t>(node_nz.begin() + N, node_nz.end()), false);
  Pod bad;
  bad.containers = {req({{"cpu", "abc"}})};
  std::vector<const Pod*> bad_pend = {&bad};
  printf("\"bad\": %d}\n", BatchSchedulingPlugin::PackNonZero({}, bad_pend, nullptr, &pod_nz).ok() ? 0 : 1);
  return 0;
}

struct Cluster {
  std::vector<Node> nodes;
  std::vector<Pod> bound;   // one pod per node carrying the node's requests
  std::vector<NodeInfo> infos;
  std::vector<PodGroup> groups;
  std::vector<Pod> pending;
};

static void set_node(Cluster& c, int i, const std::string& cpu_used, const std::string& mem_used, int num_pods) {
  c.infos[i].requested = {{"cpu", cpu_used}, {"memory", mem_used}};
  c.infos[i].num_pods = num_pods;
  Container k;
  k.requests = c.infos[i].requested;
  c.bound[i].containers = {k};
}

static Cluster make_cluster() {
  Cluster c;
  c.nodes.resize(3);
  c.bound.resize(3);
  c.infos.resize(3);
  for (int i = 0; i < 3; ++i) {
    c.nodes[i].name = "node-" + std::to_string(i);
    c.nodes[i].allocatable = {{"cpu", "8"}, {"memory", "32Gi"}, {"ephemeral-storage", "500Gi"}, {"pods", "110"}};
    c.infos[i].node = &c.nodes[i];
    c.bound[i].ns = "default"; c.bound[i].name = "bound-" + std::to_string(i); c.bound[i].uid = "bound-uid-" + std::to_string(i);
    c.infos[i].pods = {&c.bound[i]};
  }
  // node-0: most pod slots left (the min-residual best_node); node-1: least used (LeastAllocated);
  // node-2: fullest in both resources (MostAllocated)
  set_node(c, 0, "6", "4Gi", 10);
  set_node(c, 1, "1", "4Gi", 50);
  set_node(c, 2, "4", "16Gi", 80);
  c.groups.resize(1);
  c.groups[0].ns = "default"; c.groups[0].name = "pg"; c.groups[0].min_member = 1;
  c.pending.resize(2);
  for (int i = 0; i < 2; ++i) {
    Pod& p = c.pending[i];
    p.ns = "default"; p.name = "pod-" + std::to_string(i); p.uid = "uid-" + std::to_string(i);
    p.labels[kPodGroupLabel] = "pg";
    Container k;
    k.requests = {{"cpu", "500m"}, {"memory", "1Gi"}};
    p.containers = {k};
    p.queue_ts_ns = i;
  }
  c.pending[1].containers[0].requests = {{"cpu", "64"}};   // fits nowhere: an empty list
  return c;
}

static void print_plugin(BatchSchedulingPlugin& pl, bool last) {
  printf("{\"best\": %d, \"feasible\": %u, \"nodes\": [", pl.best_nodes()[0], pl.feasible_counts()[0]);
  const auto top = pl.PriorityNodes("uid-0");
  for (size_t j = 0; j < top.size(); ++j) printf("%s[\"%s\", %lld]", j ? ", " : "", top[j].first.c_str(), (long long)top[j].second);
  printf("], \"empty\": %zu, \"unknown\": %zu}%s", pl.PriorityNodes("uid-1").size(), pl.PriorityNodes("nope").size(),
         last ? "" : ", ");
}

static int cmd_round() {
  Cluster c = make_cluster();
  BatchSchedulingPlugin least(0, 0, BS_OUT_FIT_BITMAP, 0, 3), most(0, 0, BS_OUT_FIT_BITMAP, 0, 3);
  most.SetScoreWeights(0, 1, 0);
  std::vector<const NodeInfo*> snap;
  for (auto& ni : c.infos) snap.push_back(&ni);
  std::vector<const Pod*> pend;
  for (auto& p : c.pending) pend.push_back(&p);
  for (BatchSchedulingPlugin* pl : {&least, &most}) {
    pl->SetPodGroup(c.groups[0]);
    Status st = pl->BeginRound(snap, pend, 1000000000ll);
    if (!st.ok()) { fprintf(stderr, "round failed: %s\n", st.message.c_str()); return 1; }
  }
  printf("{\"begin\": [");
  print_plugin(least, false);
  print_plugin(most, true);
  // node-1 fills up with cpu: the LeastAllocated pick moves to node-2
  set_node(c, 1, "7", "4Gi", 50);
  std::vector<std::pair<uint32_t, const NodeInfo*>> changed = {{1u, &c.infos[1]}};
  for (BatchSchedulingPlugin* pl : {&least, &most}) {
    Status st = pl->UpdateRound(changed, {}, 2000000000ll);
    if (!st.ok()) { fprintf(stderr, "update failed: %s\n", st.message.c_str()); return 1; }
  }
  printf("], \"update\": [");
  print_plugin(least, false);
  print_plugin(most, true);
  BatchSchedulingPlugin unequal(0, 0, BS_OUT_FIT_BITMAP, 4, 3);
  const Status st = unequal.BeginRound(snap, pend, 1000000000ll);
  printf("], \"unequal_k_fails\": %d}\n", st.ok() ? 0 : 1);
  return 0;
}

int main(int argc, char** argv) {
  if (argc >= 2 && !strcmp(argv[1], "pack")) return cmd_pack();
  if (argc >= 2 && !strcmp(argv[1], "round")) return cmd_round();
  fprintf(stderr, "usage: %s pack | round\n", argv[0]);
  return 2;
}
