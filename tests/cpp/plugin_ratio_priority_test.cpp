// plugin_ratio_priority_test.cpp — SetRatioPriority through BatchSchedulingPlugin, printed as JSON for
// tests/test_gpu_ratio_priority.py (GPU).  Two nodes with 8 GPUs each (node-1 already uses 4) and two pending pods of
// 2 GPUs, in two rounds whose scalar resources come in different orders (round 1: example.com/foo is lane 4 and
// nvidia.com/gpu lane 5; round 2: the other way round).  The ratio setting bin-packs by GPU with `pods` and an unknown
// name in the absent weight.  Each round's PriorityNodes and ReplayQueue(kPriority) are compared with an engine built
// from the round's packed tables and given the expected lane weights and the scores multiplied by 10 directly.
#include <cstdio>
#include <map>
#include <string>
#include <utility>
#include <vector>

#include "../../batch-scheduler_b200/csrc/plugin.hpp"

using namespace bsched;

static void print_strs(const char* key, const std::vector<std::string>& v) {
  printf("\"%s\": [", key);
  for (size_t i = 0; i < v.size(); ++i) printf("%s\"%s\"", i ? ", " : "", v[i].c_str());
  printf("], ");
}
static void print_ints(const char* key, const std::vector<long long>& v, const char* tail) {
  printf("\"%s\": [", key);
  for (size_t i = 0; i < v.size(); ++i) printf("%s%lld", i ? ", " : "", v[i]);
  printf("]%s", tail);
}

static int fail(const char* what, int rc) {
  fprintf(stderr, "%s failed: %d\n", what, rc);
  return 1;
}

int main() {
  const uint32_t K = 2;
  std::vector<Node> nodes(2);
  std::vector<NodeInfo> infos(2);
  for (int i = 0; i < 2; ++i) {
    nodes[i].name = "node-" + std::to_string(i);
    infos[i].node = &nodes[i];
  }
  // the key must be in requested for a scalar request to fit (singleNodeResource, core.go:662-666)
  infos[0].requested = {{"nvidia.com/gpu", "0"}, {"example.com/foo", "0"}};
  infos[1].requested = {{"nvidia.com/gpu", "4"}, {"example.com/foo", "0"}};
  std::vector<Pod> pending(2);
  for (int i = 0; i < 2; ++i) {
    Pod& p = pending[i];
    p.ns = "default"; p.name = "pod-" + std::to_string(i); p.uid = "uid-" + std::to_string(i);
    Container k;
    k.requests = {{"cpu", "1"}, {"memory", "1Gi"}, {"nvidia.com/gpu", "2"}};
    p.containers = {k};
    p.queue_ts_ns = i;
  }
  std::vector<const NodeInfo*> snap = {&infos[0], &infos[1]};
  std::vector<const Pod*> pend = {&pending[0], &pending[1]};

  BatchSchedulingPlugin pl(0, 0, BS_OUT_FIT_BITMAP, 0, K);
  // 0..10 policy units: bin-pack
  const std::vector<std::pair<uint32_t, uint32_t>> shape = {{0, 0}, {100, 10}};
  const Status st0 = pl.SetRatioPriority(1, shape, {{"nvidia.com/gpu", 3}, {"pods", 1}, {"example.com/unknown", 2}});
  if (!st0.ok()) { fprintf(stderr, "%s\n", st0.message.c_str()); return 1; }
  const uint32_t util[2] = {0, 100}, score[2] = {0, 100};

  printf("{\"rounds\": [");
  for (int round = 0; round < 2; ++round) {
    const ResourceList base = {{"cpu", "16"}, {"memory", "64Gi"}, {"pods", "110"}};
    ResourceList a0 = base, a1 = base;
    if (round == 0) {
      a0.insert(a0.end(), {{"example.com/foo", "4"}, {"nvidia.com/gpu", "8"}});
      a1.insert(a1.end(), {{"nvidia.com/gpu", "8"}, {"example.com/foo", "4"}});
    } else {
      a0.insert(a0.end(), {{"nvidia.com/gpu", "8"}, {"example.com/foo", "4"}});
      a1.insert(a1.end(), {{"example.com/foo", "4"}, {"nvidia.com/gpu", "8"}});
    }
    nodes[0].allocatable = a0;
    nodes[1].allocatable = a1;
    const Status st = pl.BeginRound(snap, pend, 1000000000ll * (round + 1));
    if (!st.ok()) { fprintf(stderr, "round failed: %s\n", st.message.c_str()); return 1; }
    std::vector<BatchSchedulingPlugin::ReplayDecision> dec;
    const Status rs = pl.ReplayQueue(&dec, BatchSchedulingPlugin::ReplayNodeChoice::kPriority);
    if (!rs.ok()) { fprintf(stderr, "replay failed: %s\n", rs.message.c_str()); return 1; }

    // the same round on an engine called directly, with the lane weights worked out here
    const PackedSnapshot& ps = pl.packed();
    const uint32_t L = ps.lanes;
    int gpu_lane = -1;
    for (size_t k = 0; k < ps.scalar_names.size(); ++k)
      if (ps.scalar_names[k] == "nvidia.com/gpu") gpu_lane = (int)(4 + k);
    std::vector<uint32_t> lane_w(L, 0);
    lane_w[gpu_lane] = 3;
    bs_config cfg{0, L, BS_OUT_PRIORITY, K};
    bs_engine* e = nullptr;
    int rc = bs_create(&cfg, &e);
    if (rc) return fail("bs_create", rc);
    const bs_node_table nt = ps.node_table();
    const bs_group_table gt = ps.group_table();
    const bs_pod_table pt = ps.pod_table();
    std::vector<int64_t> node_nz, pod_nz;
    BatchSchedulingPlugin::PackNonZero(snap, pend, &node_nz, &pod_nz);
    if ((rc = bs_upload_nodes(e, &nt)) || (rc = bs_upload_groups(e, &gt)) || (rc = bs_upload_pods(e, &pt)) ||
        (rc = bs_upload_node_nonzero(e, 2, node_nz.data())) || (rc = bs_upload_pod_nonzero(e, 2, pod_nz.data())) ||
        (rc = bs_set_ratio_priority(e, 1, 2, util, score, L, lane_w.data(), 1 + 2)))
      return fail("engine setup", rc);
    bs_results res{};
    if ((rc = bs_evaluate(e, &res))) return fail("bs_evaluate", rc);
    std::vector<int32_t> en(2 * K);
    std::vector<int64_t> es(2 * K);
    if ((rc = bs_fetch_priority_rows(e, 0, 2, en.data(), es.data()))) return fail("bs_fetch_priority_rows", rc);
    std::vector<uint32_t> order = pl.queue_order();
    std::vector<uint8_t> pf(2), ready(2);
    std::vector<int32_t> rn(2);
    bs_replay_result rr{};
    rr.prefilter = pf.data(); rr.node = rn.data(); rr.ready = ready.data();
    if ((rc = bs_replay_priority(e, order.data(), 2, &rr, nullptr))) return fail("bs_replay_priority", rc);
    bs_destroy(e);

    std::vector<std::string> pn, enames;
    std::vector<long long> psc, esc, prep, erep;
    for (auto& kv : pl.PriorityNodes("uid-0")) { pn.push_back(kv.first); psc.push_back(kv.second); }
    for (uint32_t k = 0; k < K && en[k] >= 0; ++k) { enames.push_back(nodes[en[k]].name); esc.push_back(es[k]); }
    for (auto& d : dec) prep.push_back(d.node);
    for (int32_t n : rn) erep.push_back(n);
    printf("%s{\"gpu_lane\": %d, ", round ? ", " : "", gpu_lane);
    print_strs("plugin_nodes", pn);
    print_strs("engine_nodes", enames);
    print_ints("plugin_scores", psc, ", ");
    print_ints("engine_scores", esc, ", ");
    print_ints("plugin_replay", prep, ", ");
    print_ints("engine_replay", erep, "}");
  }
  const Status bad = pl.SetRatioPriority(1, {{50, 5}, {50, 6}}, {});
  printf("], \"invalid_shape_fails\": %d}\n", bad.ok() ? 0 : 1);
  return 0;
}
