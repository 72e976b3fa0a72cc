// plugin_preempt_host_ports_test.cpp — Preempt, PreemptAll and PreemptQueue of BatchSchedulingPlugin under the
// PodFitsHostPorts filter (SetHostPortFilterInPreemption), as JSON for tests/test_plugin_preempt_host_ports.py.
//   run   (GPU) two full nodes whose bound pods hold host ports, three pending pods asking for ports; the three calls
//         with the filter off, with the filter and the option on, and with the filter on and the option off; and the
//         bound masks PackHostPorts(..., bound = true) packs
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

static ContainerPort port(const char* ip, int32_t p) {
  ContainerPort cp;
  cp.host_ip = ip;
  cp.host_port = p;
  cp.container_port = p;
  return cp;
}

static Pod make_pod(const std::string& name, const char* cpu, int32_t prio, int64_t start,
                    std::vector<ContainerPort> ports) {
  Pod p;
  p.ns = "ns"; p.name = name; p.uid = "uid-" + name;
  Container c;
  c.requests = {{"cpu", cpu}};
  c.ports = std::move(ports);
  p.containers = {c};
  p.priority = prio;
  p.start_ns = start;
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

static int cmd_run() {
  // node-0 and node-1: 4 cpus, fully requested by 2-cpu online pods.  node-0 holds a (prio 0, start 50, 0.0.0.0:22)
  // and b (prio 0, start 100, no port); node-1 holds c (prio 0, start 100, 10.0.0.1:22) and d (prio 100, start 0,
  // 0.0.0.0:8080).  Pending, 1 cpu and priority 10 each, in queue order: p (0.0.0.0:22), q (0.0.0.0:8080), r (:22).
  std::vector<Node> nodes(2);
  std::vector<NodeInfo> infos(2);
  Pod a = make_pod("a", "2", 0, 50, {port("", 22)}), b = make_pod("b", "2", 0, 100, {});
  Pod c = make_pod("c", "2", 0, 100, {port("10.0.0.1", 22)}), d = make_pod("d", "2", 100, 0, {port("0.0.0.0", 8080)});
  for (int i = 0; i < 2; ++i) {
    nodes[i].name = "node-" + std::to_string(i);
    nodes[i].allocatable = {{"cpu", "4"}, {"memory", "8Gi"}, {"pods", "110"}};
    infos[i].node = &nodes[i];
    infos[i].requested = {{"cpu", "4"}};
  }
  infos[0].pods = {&a, &b};
  infos[1].pods = {&c, &d};
  for (auto& ni : infos) {
    ni.num_pods = (int32_t)ni.pods.size();
    for (const Pod* p : ni.pods) ni.used_ports.insert(ni.used_ports.end(), p->containers[0].ports.begin(),
                                                      p->containers[0].ports.end());
  }
  Pod p = make_pod("p", "1", 10, 0, {port("", 22)}), q = make_pod("q", "1", 10, 0, {port("", 8080)});
  Pod r = make_pod("r", "1", 10, 0, {port("0.0.0.0", 22)});
  p.queue_ts_ns = 1; q.queue_ts_ns = 2; r.queue_ts_ns = 3;
  std::vector<const NodeInfo*> snap = {&infos[0], &infos[1]};
  std::vector<const Pod*> pend = {&p, &q, &r};
  printf("{");
  {
    PackedHostPorts pk;
    Status st = BatchSchedulingPlugin::PackHostPorts(snap, pend, &pk, true);
    printf("\"packed\": {\"ok\": %s, \"entries\": [", st.ok() ? "true" : "false");
    for (size_t k = 0; k < pk.port.size(); ++k)
      printf("%s[%s, %s, %d]", k ? ", " : "", json_str(pk.ips[pk.ip[k]]).c_str(),
             json_str(pk.protocols[pk.protocol[k]]).c_str(), pk.port[k]);
    printf("], \"used\": [");
    for (size_t k = 0; k < pk.used.size(); ++k) printf("%s%llu", k ? ", " : "", (unsigned long long)pk.used[k]);
    printf("], \"bound\": [");
    for (size_t k = 0; k < pk.bound.size(); ++k) printf("%s%llu", k ? ", " : "", (unsigned long long)pk.bound[k]);
    printf("]}");
  }
  const char* modes[] = {"off", "on", "refused"};
  for (int m = 0; m < 3; ++m) {
    BatchSchedulingPlugin plugin(0, 0, BS_OUT_FIT_BITMAP);
    plugin.SetHostPortFilter(m != 0);
    plugin.SetHostPortFilterInPreemption(m != 2);
    Status st = plugin.BeginRound(snap, pend, 1000000000ll);
    if (!st.ok()) { fprintf(stderr, "round failed: %s\n", st.message.c_str()); return 1; }
    printf(", %s: {", json_str(modes[m]).c_str());
    std::vector<BatchSchedulingPlugin::Preemption> v;
    st = plugin.PreemptAll(&v);
    print_list("all", st, v);
    printf(", ");
    st = plugin.PreemptQueue(&v, false);
    print_list("queue", st, v);
    std::string node;
    std::vector<std::string> victims;
    st = plugin.Preempt("uid-r", &node, &victims);
    printf(", \"preempt_r\": {\"ok\": %s, \"message\": %s, \"node\": %s, \"victims\": [", st.ok() ? "true" : "false",
           json_str(st.message).c_str(), json_str(node).c_str());
    for (size_t k = 0; k < victims.size(); ++k) printf("%s%s", k ? ", " : "", json_str(victims[k]).c_str());
    printf("]}}");
  }
  printf("}\n");
  return 0;
}

int main(int argc, char** argv) {
  if (argc >= 2 && !strcmp(argv[1], "run")) return cmd_run();
  fprintf(stderr, "usage: %s run\n", argv[0]);
  return 2;
}
