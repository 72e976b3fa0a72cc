// plugin_preempt_walk_test.cpp — BatchSchedulingPlugin::PreemptQueue (bs_preempt_walk), as JSON for
// tests/test_plugin_preempt_walk.py.
//   walk   (GPU) the two-node scenario of tests/preempt_walk_cases.py through a round: PreemptQueue with and without
//          gang units, PreemptAll and Preempt on the same pods, and a group whose pending pods differ in priority
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

static Pod make_pod(const std::string& name, const char* cpu, int32_t prio, const char* group, int64_t start) {
  Pod p;
  p.ns = "ns"; p.name = name; p.uid = "uid-" + name;
  Container c;
  c.requests = {{"cpu", cpu}};
  p.containers = {c};
  p.priority = prio;
  p.start_ns = start;
  if (group) p.labels[kPodGroupLabel] = group;
  return p;
}

static void print_list(const char* key, const Status& st, const std::vector<BatchSchedulingPlugin::Preemption>& v) {
  printf("%s: {\"ok\": %s, \"message\": %s, \"entries\": [", json_str(key).c_str(), st.ok() ? "true" : "false",
         json_str(st.message).c_str());
  for (size_t i = 0; i < v.size(); ++i) {
    printf("%s[%s, %s, [", i ? ", " : "", json_str(v[i].uid).c_str(), json_str(v[i].node).c_str());
    for (size_t k = 0; k < v[i].victims.size(); ++k) printf("%s%s", k ? ", " : "", json_str(v[i].victims[k]).c_str());
    printf("]]");
  }
  printf("]}");
}

// bs_preempt_walk called directly on the pending rows of `v`'s uids in `v`'s order, printed as `v` is: node names and
// victim uids.  Pending row i is pend[i] (BeginRound's order).
static void print_direct(const char* key, BatchSchedulingPlugin& plugin, const std::vector<const Pod*>& pend,
                         const std::vector<BatchSchedulingPlugin::Preemption>& v, uint32_t flags) {
  std::vector<uint32_t> rows;
  for (const auto& pr : v)
    for (uint32_t i = 0; i < pend.size(); ++i)
      if (pend[i]->uid == pr.uid) rows.push_back(i);
  const uint32_t n = (uint32_t)rows.size();
  std::vector<int32_t> node(n + 1);
  std::vector<uint32_t> nv(n + 1), cand(n + 1), off(n + 1), vict(plugin.bound().n + 1);
  bs_preempt_result r{node.data(), nv.data(), cand.data(), off.data(), vict.data(), plugin.bound().n, 0};
  const int rc = bs_preempt_walk(plugin.engine(), rows.data(), n, flags, &r, nullptr, nullptr);
  printf("%s: {\"rc\": %d, \"entries\": [", json_str(key).c_str(), rc);
  for (uint32_t i = 0; i < n && rc == BS_OK; ++i) {
    printf("%s[%s, %s, [", i ? ", " : "", json_str(pend[rows[i]]->uid).c_str(),
           json_str(node[i] >= 0 ? "node-" + std::to_string(node[i]) : std::string()).c_str());
    for (uint32_t k = off[i]; k < off[i + 1]; ++k)
      printf("%s%s", k > off[i] ? ", " : "", json_str(plugin.bound().pods[vict[k]]->uid).c_str());
    printf("]]");
  }
  printf("]}");
}

static int cmd_walk() {
  // node-0 and node-1: 4 cpus, fully requested by 2-cpu pods of the Pending group "h": node-0 holds a (prio 0, start
  // 50) and b (prio 0, start 100), node-1 d (prio 5) and c (prio 0, start 100).  node-2 and node-3 have 2 free cpus
  // each and no pods: no preemptor fits or preempts there, but the group's cluster check passes on their sum.
  std::vector<Node> nodes(4);
  std::vector<NodeInfo> infos(4);
  Pod a = make_pod("a", "2", 0, "h", 50), b = make_pod("b", "2", 0, "h", 100);
  Pod d = make_pod("d", "2", 5, "h", 0), c = make_pod("c", "2", 0, "h", 100);
  for (int i = 0; i < 4; ++i) {
    nodes[i].name = "node-" + std::to_string(i);
    nodes[i].allocatable = {{"cpu", "4"}, {"memory", "8Gi"}, {"pods", "110"}};
    infos[i].node = &nodes[i];
    infos[i].requested = {{"cpu", i < 2 ? "4" : "2"}};
  }
  infos[0].pods = {&a, &b};
  infos[1].pods = {&d, &c};
  for (auto& ni : infos) ni.num_pods = (int32_t)ni.pods.size();
  // preemptors (3 cpus, priority 10): g1 g2 g3 of the Pending group "g", the online q between them in queue time
  Pod g1 = make_pod("g1", "3", 10, "g", 0), q = make_pod("q", "3", 10, nullptr, 0);
  Pod g2 = make_pod("g2", "3", 10, "g", 0), g3 = make_pod("g3", "3", 10, "g", 0);
  g1.queue_ts_ns = 1; q.queue_ts_ns = 2; g2.queue_ts_ns = 3; g3.queue_ts_ns = 4;
  auto run = [&](int32_t g3_prio, bool first) {
    g3.priority = g3_prio;
    BatchSchedulingPlugin plugin(0, 0, BS_OUT_FIT_BITMAP);
    for (const char* name : {"h", "g"}) {
      PodGroup pg;
      pg.ns = "ns"; pg.name = name; pg.min_member = 1; pg.phase = "Pending";
      plugin.SetPodGroup(pg);
    }
    std::vector<const NodeInfo*> snap = {&infos[0], &infos[1], &infos[2], &infos[3]};
    std::vector<const Pod*> pend = {&g1, &q, &g2, &g3};
    Status st = plugin.BeginRound(snap, pend, 1000000000ll);
    if (!st.ok()) { fprintf(stderr, "round failed: %s\n", st.message.c_str()); return 1; }
    std::vector<BatchSchedulingPlugin::Preemption> v;
    if (first) {
      printf("{\"bound\": %u, ", plugin.bound().n);
      st = plugin.PreemptAll(&v);
      print_list("all", st, v);
      printf(", ");
      st = plugin.PreemptQueue(&v, false);
      print_list("queue", st, v);
      printf(", ");
      print_direct("queue_direct", plugin, pend, v, 0);
      printf(", \"first\": ");
      std::string node;
      std::vector<std::string> victims;
      st = plugin.Preempt(v.empty() ? "" : v[0].uid, &node, &victims);
      printf("[%s, [", json_str(st.ok() ? node : "error").c_str());
      for (size_t k = 0; k < victims.size(); ++k) printf("%s%s", k ? ", " : "", json_str(victims[k]).c_str());
      printf("]], ");
      st = plugin.PreemptQueue(&v, true);
      print_list("gang", st, v);
      printf(", ");
      print_direct("gang_direct", plugin, pend, v, BS_PREEMPT_GANG);
    } else {
      printf(", ");
      st = plugin.PreemptQueue(&v, true);
      print_list("mixed_gang", st, v);
      printf(", ");
      st = plugin.PreemptQueue(&v, false);
      print_list("mixed_queue", st, v);
      printf("}\n");
    }
    return 0;
  };
  if (run(10, true)) return 1;
  return run(9, false);
}

int main(int argc, char** argv) {
  if (argc >= 2 && !strcmp(argv[1], "walk")) return cmd_walk();
  fprintf(stderr, "usage: %s walk\n", argv[0]);
  return 2;
}
