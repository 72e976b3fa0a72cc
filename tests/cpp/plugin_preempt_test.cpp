// plugin_preempt_test.cpp — preemption through BatchSchedulingPlugin, as JSON for tests/test_plugin_preempt.py.
//   pack   (CPU) PackBoundPods: Requests not Limits, the group label and Status.Phase -> gid / locked flag, errors
//   gang   (GPU) a scripted gang scenario: RemovePod messages, Preempt / PreemptAll, and a delta round that locks a gang
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

static int cmd_pack() {
  PackedSnapshot ctx;
  ctx.lanes = 5;
  ctx.scalar_names = {"nvidia.com/gpu"};
  Pod a = make_pod("a", "1", 3, nullptr, 7);   // Requests 1 cpu, Limits 4 cpu and a GPU request
  a.containers[0].has_limits = true;
  a.containers[0].limits = {{"cpu", "4"}};
  a.containers[0].requests.push_back({"nvidia.com/gpu", "1"});
  a.containers[0].requests.push_back({"pods", "5"});   // lane 3 is not a pod's request
  Pod b = make_pod("b", "500m", -4, "pend", 8);
  Pod c = make_pod("c", "2", 0, "run", 9);
  Pod d = make_pod("d", "2", 0, "sched", 9);
  Pod e = make_pod("e", "2", 0, "gone", 9);
  NodeInfo n0, n1;
  n0.pods = {&a, &b};
  n1.pods = {&c, &d, &e};
  const std::unordered_map<std::string, uint32_t> rows = {{"ns/pend", 0}, {"ns/run", 1}, {"ns/sched", 2}};
  const std::vector<uint8_t> locked = {0, 1, 1};
  PackedBound out;
  Status st = BatchSchedulingPlugin::PackBoundPods(ctx, {&n0, &n1}, rows, locked, &out);
  printf("{\"ok\": %s, \"n\": %u, \"node\": [", st.ok() ? "true" : "false", out.n);
  for (uint32_t k = 0; k < out.n; ++k) printf("%s%u", k ? ", " : "", out.node[k]);
  printf("], \"req\": [");
  for (uint32_t d2 = 0; d2 < out.lanes; ++d2) {
    printf("%s[", d2 ? ", " : "");
    for (uint32_t k = 0; k < out.n; ++k) printf("%s%lld", k ? ", " : "", (long long)out.req[(size_t)d2 * out.n + k]);
    printf("]");
  }
  printf("], \"req_present\": [");
  for (uint32_t k = 0; k < out.n; ++k) printf("%s%u", k ? ", " : "", out.req_present[k]);
  printf("], \"gid\": [");
  for (uint32_t k = 0; k < out.n; ++k) printf("%s%d", k ? ", " : "", out.gid[k]);
  printf("], \"flags\": [");
  for (uint32_t k = 0; k < out.n; ++k) printf("%s%u", k ? ", " : "", out.flags[k]);
  printf("], \"priority\": [");
  for (uint32_t k = 0; k < out.n; ++k) printf("%s%d", k ? ", " : "", out.priority[k]);
  printf("], \"start\": [");
  for (uint32_t k = 0; k < out.n; ++k) printf("%s%lld", k ? ", " : "", (long long)out.start_ns[k]);
  // errors: a scalar resource the round has no lane for, a malformed quantity
  Pod f = make_pod("f", "1", 0, nullptr, 0);
  f.containers[0].requests.push_back({"example.com/fpga", "1"});
  Pod g = make_pod("g", "1x", 0, nullptr, 0);
  NodeInfo n2, n3;
  n2.pods = {&f};
  n3.pods = {&g};
  const Status e1 = BatchSchedulingPlugin::PackBoundPods(ctx, {&n2}, rows, locked, &out);
  const Status e2 = BatchSchedulingPlugin::PackBoundPods(ctx, {&n3}, rows, locked, &out);
  printf("], \"errors\": [%s, %s]}\n", json_str(e1.ok() ? "" : e1.message).c_str(),
         json_str(e2.ok() ? "" : e2.message).c_str());
  return 0;
}

static void print_preempt(BatchSchedulingPlugin& plugin, const std::string& uid, bool last) {
  std::string node;
  std::vector<std::string> victims;
  const Status st = plugin.Preempt(uid, &node, &victims);
  printf("%s: [%s, ", json_str(uid).c_str(), json_str(st.ok() ? node : "error: " + st.message).c_str());
  printf("[");
  for (size_t k = 0; k < victims.size(); ++k) printf("%s%s", k ? ", " : "", json_str(victims[k]).c_str());
  printf("]]%s", last ? "" : ", ");
}

static void print_remove(BatchSchedulingPlugin& plugin, const Pod& p, const Pod& v, bool last) {
  const Status st = plugin.RemovePod(p, v);
  printf("[%d, %s]%s", st.code, json_str(st.message).c_str(), last ? "" : ", ");
}

static void print_all(BatchSchedulingPlugin& plugin) {
  std::vector<BatchSchedulingPlugin::Preemption> all;
  const Status st = plugin.PreemptAll(&all);
  printf("\"all_ok\": %s, \"all\": [", st.ok() ? "true" : "false");
  for (size_t i = 0; i < all.size(); ++i) {
    printf("%s[%s, %s, [", i ? ", " : "", json_str(all[i].uid).c_str(), json_str(all[i].node).c_str());
    for (size_t k = 0; k < all[i].victims.size(); ++k) printf("%s%s", k ? ", " : "", json_str(all[i].victims[k]).c_str());
    printf("]]");
  }
  printf("]");
}

static int cmd_gang() {
  // three full nodes with 4 cpus: node-0 (zone=a) runs the Pending gang "pend" (priority 50), node-1 (zone=a) the
  // Running gang "run" (priority 1), node-2 an online pod (priority 1)
  std::vector<Node> nodes(3);
  std::vector<NodeInfo> infos(3);
  Pod pa = make_pod("pend-a", "2", 50, "pend", 1), pb = make_pod("pend-b", "2", 50, "pend", 2);
  Pod ra = make_pod("run-a", "2", 1, "run", 1), rb = make_pod("run-b", "2", 1, "run", 2);
  Pod on = make_pod("online", "4", 1, nullptr, 1);
  for (int i = 0; i < 3; ++i) {
    nodes[i].name = "node-" + std::to_string(i);
    nodes[i].allocatable = {{"cpu", "4"}, {"memory", "8Gi"}, {"pods", "110"}};
    if (i < 2) nodes[i].labels = {{"zone", "a"}};
    infos[i].node = &nodes[i];
    infos[i].requested = {{"cpu", "4"}};
  }
  infos[0].pods = {&pa, &pb};
  infos[1].pods = {&ra, &rb};
  infos[2].pods = {&on};
  for (auto& ni : infos) ni.num_pods = (int32_t)ni.pods.size();
  // preemptors (priority 100, 2 cpus): online P1; online P3 restricted to zone=a; offline P2 of the Pending gang "other"
  Pod p1 = make_pod("p1", "2", 100, nullptr, 0), p3 = make_pod("p3", "2", 100, nullptr, 0);
  p3.node_selector = {{"zone", "a"}};
  Pod p2 = make_pod("p2", "2", 100, "other", 0);
  BatchSchedulingPlugin plugin(0, 0, BS_OUT_FIT_BITMAP);
  auto group = [&](const char* name, const char* phase, uint32_t min_member) {
    PodGroup pg;
    pg.ns = "ns"; pg.name = name; pg.min_member = min_member; pg.phase = phase;
    plugin.SetPodGroup(pg);
  };
  group("pend", "Pending", 2);
  group("run", "Running", 2);
  group("other", "Pending", 1);
  std::vector<const NodeInfo*> snap = {&infos[0], &infos[1], &infos[2]};
  std::vector<const Pod*> pend = {&p1, &p2, &p3};
  Status st = plugin.BeginRound(snap, pend, 1000000000ll);
  if (!st.ok()) { fprintf(stderr, "round failed: %s\n", st.message.c_str()); return 1; }
  printf("{\"bound\": %u, \"preempt\": {", plugin.bound().n);
  print_preempt(plugin, p1.uid, false);
  print_preempt(plugin, p2.uid, false);
  print_preempt(plugin, p3.uid, true);
  printf("}, \"remove\": [");
  print_remove(plugin, p1, pa, false);
  print_remove(plugin, p1, ra, false);
  print_remove(plugin, p1, on, false);
  print_remove(plugin, p2, on, false);
  print_remove(plugin, p2, pa, false);
  print_remove(plugin, p2, ra, true);
  printf("], ");
  print_all(plugin);
  // the Pending gang starts running: a group update locks its pods, P3 has nowhere left to go
  group("pend", "Running", 2);
  st = plugin.UpdateRound({}, {"ns/pend"}, 2000000000ll);
  if (!st.ok()) { fprintf(stderr, "update failed: %s\n", st.message.c_str()); return 1; }
  printf(", \"after\": {");
  print_preempt(plugin, p3.uid, false);
  print_preempt(plugin, p1.uid, true);
  printf("}, \"unknown\": ");
  std::string node;
  printf("%s}\n", json_str(plugin.Preempt("no-such-uid", &node, nullptr).ok() ? "ok" : "error").c_str());
  return 0;
}

int main(int argc, char** argv) {
  if (argc >= 2 && !strcmp(argv[1], "pack")) return cmd_pack();
  if (argc >= 2 && !strcmp(argv[1], "gang")) return cmd_gang();
  fprintf(stderr, "usage: %s pack|gang\n", argv[0]);
  return 2;
}
