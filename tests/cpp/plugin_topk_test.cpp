// plugin_topk_test.cpp — BatchSchedulingPlugin created with a top-K list length: after BeginRound and after an
// UpdateRound, prints for every pending pod TopNodes(uid) and the engine's own rows (bs_fetch_topk_rows), as JSON
// for tests/test_gpu_topk.py.
//   topk <K>   (GPU)
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../batch-scheduler_b200/csrc/plugin.hpp"

using namespace bsched;

static void print_round(BatchSchedulingPlugin& plugin, const std::vector<Pod>& pods, uint32_t K, bool last) {
  const uint32_t P = (uint32_t)pods.size();
  std::vector<int32_t> nodes((size_t)P * K);
  std::vector<int64_t> scores((size_t)P * K);
  const int rc = bs_fetch_topk_rows(plugin.engine(), 0, P, nodes.data(), scores.data());
  printf("{\"rc\": %d, \"feasible\": [", rc);
  for (uint32_t i = 0; i < P; ++i) printf("%s%u", i ? ", " : "", plugin.feasible_counts()[i]);
  printf("], \"best\": [");
  for (uint32_t i = 0; i < P; ++i) printf("%s%d", i ? ", " : "", plugin.best_nodes()[i]);
  printf("], \"rows_node\": [");
  for (size_t i = 0; i < nodes.size(); ++i) printf("%s%d", i ? ", " : "", nodes[i]);
  printf("], \"rows_score\": [");
  for (size_t i = 0; i < scores.size(); ++i) printf("%s%lld", i ? ", " : "", (long long)scores[i]);
  printf("], \"top\": [");
  for (uint32_t i = 0; i < P; ++i) {
    printf("%s[", i ? ", " : "");
    const auto top = plugin.TopNodes(pods[i].uid);
    for (size_t j = 0; j < top.size(); ++j) printf("%s[\"%s\", %lld]", j ? ", " : "", top[j].first.c_str(), (long long)top[j].second);
    printf("]");
  }
  printf("], \"unknown\": %zu}%s\n", plugin.TopNodes("no-such-uid").size(), last ? "" : ",");
}

static int cmd_topk(uint32_t K) {
  const int N = 300, P = 100, G = 10;
  std::vector<Node> nodes(N);
  std::vector<NodeInfo> infos(N);
  for (int i = 0; i < N; ++i) {
    nodes[i].name = "node-" + std::to_string(i);
    // every fourth node identical to the one before it: equal scores, ordered by snapshot index
    const int k = i % 4 == 3 ? i - 1 : i;
    nodes[i].allocatable = {{"cpu", std::to_string(4 + k % 7 * 4)}, {"memory", std::to_string(16 + k % 5 * 8) + "Gi"},
                            {"ephemeral-storage", "500Gi"}, {"pods", "110"}};
    infos[i].node = &nodes[i];
    infos[i].requested = {{"cpu", std::to_string(250 * (k % 13)) + "m"}, {"memory", std::to_string(k % 9) + "Gi"}};
    infos[i].num_pods = k % 40;
  }
  std::vector<PodGroup> groups(G);
  for (int g = 0; g < G; ++g) {
    groups[g].ns = "default"; groups[g].name = "pg-" + std::to_string(g); groups[g].min_member = 1 + g % 4;
    groups[g].creation_ns = 1600000000ll * 1000000000ll + g * 1000000000ll;
  }
  std::vector<Pod> pods(P);
  for (int i = 0; i < P; ++i) {
    Pod& p = pods[i];
    p.ns = "default"; p.name = "pod-" + std::to_string(i); p.uid = "uid-" + std::to_string(i);
    p.labels[kPodGroupLabel] = "pg-" + std::to_string(i % G);
    Container c; c.has_limits = true;
    // pod 7 asks for more cpu than any node has: it fits nowhere
    c.limits = {{"cpu", i == 7 ? std::string("1000") : std::to_string(500 * (1 + i % 9)) + "m"},
                {"memory", std::to_string(1 + i % 12) + "Gi"}};
    p.containers = {c};
    p.priority = i % 5; p.queue_ts_ns = i;
  }
  BatchSchedulingPlugin plugin(0, 0, BS_OUT_FIT_BITMAP, K);
  for (auto& g : groups) plugin.SetPodGroup(g);
  std::vector<const NodeInfo*> snap(N);
  std::vector<const Pod*> pend(P);
  for (int i = 0; i < N; ++i) snap[i] = &infos[i];
  for (int i = 0; i < P; ++i) pend[i] = &pods[i];
  Status st = plugin.BeginRound(snap, pend, 1000000000ll);
  if (!st.ok()) { fprintf(stderr, "round failed: %s\n", st.message.c_str()); return 1; }
  printf("[\n");
  print_round(plugin, pods, K, false);
  // a delta round: three nodes empty out (the pod-count lane holds every pair's smallest residual, so they join the
  // nodes without pods at the front of the lists), one fills up
  std::vector<std::pair<uint32_t, const NodeInfo*>> changed;
  for (int i : {5, 77, 150, 299}) {
    infos[i].requested = {{"cpu", i == 150 ? std::string("64") : std::string("0")}, {"memory", "0"}};
    infos[i].num_pods = i == 150 ? 110 : 0;
    changed.push_back({(uint32_t)i, &infos[i]});
  }
  st = plugin.UpdateRound(changed, {}, 2000000000ll);
  if (!st.ok()) { fprintf(stderr, "update failed: %s\n", st.message.c_str()); return 1; }
  print_round(plugin, pods, K, true);
  printf("]\n");
  return 0;
}

int main(int argc, char** argv) {
  if (argc >= 3 && !strcmp(argv[1], "topk")) return cmd_topk((uint32_t)atoi(argv[2]));
  fprintf(stderr, "usage: %s topk <K>\n", argv[0]);
  return 2;
}
