// plugin_replay_priority_test.cpp — ReplayQueue's node choices through BatchSchedulingPlugin, printed as JSON for
// tests/test_gpu_replay_priority.py (GPU).  Two empty nodes of 4 cpu / 8Gi and four pending pods of 500m / 1Gi outside
// any PodGroup, walked with kFirstFit, with kPriority under weights (1, 0, 1) and (0, 1, 0), and kPriority on a plugin
// created without priority_k (an error).
#include <cstdio>
#include <cstring>
#include <string>
#include <tuple>
#include <vector>

#include "../../batch-scheduler_b200/csrc/plugin.hpp"

using namespace bsched;

static void print_nodes(const char* key, const std::vector<BatchSchedulingPlugin::ReplayDecision>& d, bool last) {
  printf("\"%s\": [", key);
  for (size_t i = 0; i < d.size(); ++i) printf("%s%d", i ? ", " : "", d[i].node);
  printf("]%s", last ? "" : ", ");
}

int main() {
  std::vector<Node> nodes(2);
  std::vector<NodeInfo> infos(2);
  for (int i = 0; i < 2; ++i) {
    nodes[i].name = "node-" + std::to_string(i);
    nodes[i].allocatable = {{"cpu", "4"}, {"memory", "8Gi"}, {"pods", "110"}};
    infos[i].node = &nodes[i];
  }
  std::vector<Pod> pending(4);
  for (int i = 0; i < 4; ++i) {
    Pod& p = pending[i];
    p.ns = "default"; p.name = "pod-" + std::to_string(i); p.uid = "uid-" + std::to_string(i);
    Container k;
    k.requests = {{"cpu", "500m"}, {"memory", "1Gi"}};
    p.containers = {k};
    p.queue_ts_ns = i;
  }
  std::vector<const NodeInfo*> snap = {&infos[0], &infos[1]};
  std::vector<const Pod*> pend;
  for (auto& p : pending) pend.push_back(&p);

  using Choice = BatchSchedulingPlugin::ReplayNodeChoice;
  BatchSchedulingPlugin least(0, 0, BS_OUT_FIT_BITMAP, 0, 1), most(0, 0, BS_OUT_FIT_BITMAP, 0, 1),
      plain(0, 0, BS_OUT_FIT_BITMAP);
  most.SetScoreWeights(0, 1, 0);
  for (BatchSchedulingPlugin* pl : {&least, &most, &plain}) {
    const Status st = pl->BeginRound(snap, pend, 1000000000ll);
    if (!st.ok()) { fprintf(stderr, "round failed: %s\n", st.message.c_str()); return 1; }
  }
  std::vector<BatchSchedulingPlugin::ReplayDecision> first, spread, pack, plain_first, plain_prio;
  for (auto [pl, choice, out] : {std::make_tuple(&least, Choice::kFirstFit, &first),
                                 std::make_tuple(&least, Choice::kPriority, &spread),
                                 std::make_tuple(&most, Choice::kPriority, &pack),
                                 std::make_tuple(&plain, Choice::kFirstFit, &plain_first)}) {
    const Status st = pl->ReplayQueue(out, choice);
    if (!st.ok()) { fprintf(stderr, "replay failed: %s\n", st.message.c_str()); return 1; }
  }
  const Status err = plain.ReplayQueue(&plain_prio, Choice::kPriority);
  printf("{");
  print_nodes("first_fit", first, false);
  print_nodes("least_balanced", spread, false);
  print_nodes("most", pack, false);
  print_nodes("plain_first_fit", plain_first, false);
  printf("\"positions\": [");
  for (size_t i = 0; i < spread.size(); ++i) printf("%s%u", i ? ", " : "", spread[i].position);
  printf("], \"no_priority_k_fails\": %d, \"message\": \"%s\"}\n", err.ok() ? 0 : 1, err.message.c_str());
  return 0;
}
