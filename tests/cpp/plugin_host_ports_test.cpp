// plugin_host_ports_test.cpp — BatchSchedulingPlugin::PackHostPorts and SetHostPortFilter, printed as JSON for
// tests/test_plugin_host_ports.py.  Seeded rounds of eight nodes with used host ports and pending pods whose containers
// ask for ports over the wildcard, empty, specific and "::" ips, empty / TCP / UDP protocols and ports <= 0.  The
// program prints the objects, so that the test packs and evaluates them independently, the columns PackHostPorts made
// of them, and whether a round of 65 distinct wanted entries is refused.  With the argument "gpu" it also runs a round
// of the first scenario on the device with SetHostPortFilter(true) and prints each pending pod's FitError, ReasonCounts
// and HostPortReasonCounts; the same after UpdateNodes and after UpdateRound gave node 0 every wanted port; whether
// Preempt, PreemptAll and PreemptQueue refuse the filter; and whether ReplayQueue runs under it.
#include <cstdio>
#include <cstring>
#include <random>
#include <string>
#include <vector>

#include "../../batch-scheduler_b200/csrc/plugin.hpp"

using namespace bsched;

static std::string q(const std::string& s) { return "\"" + s + "\""; }   // the texts here need no escaping
template <class T>
static std::string jnums(const std::vector<T>& v) {
  std::string o = "[";
  for (size_t k = 0; k < v.size(); ++k) o += (k ? ", " : "") + std::to_string(v[k]);
  return o + "]";
}
static std::string jports(const std::vector<ContainerPort>& v) {
  std::string o = "[";
  for (size_t k = 0; k < v.size(); ++k)
    o += (k ? ", " : "") + std::string("[") + q(v[k].host_ip) + ", " + q(v[k].protocol) + ", " +
         std::to_string(v[k].host_port) + ", " + std::to_string(v[k].container_port) + "]";
  return o + "]";
}

struct Gen {
  std::mt19937 r;
  explicit Gen(uint32_t seed) : r(seed) {}
  uint32_t below(uint32_t n) { return r() % n; }
};
static ContainerPort random_port(Gen& g) {
  static const char* IPS[] = {"", "", "0.0.0.0", "10.0.0.1", "10.0.0.2", "::"};
  static const char* PROTOS[] = {"", "TCP", "UDP"};
  static const int32_t PORTS[] = {0, -1, 80, 443, 8080, 8080, 29500};
  ContainerPort p;
  p.host_ip = IPS[g.below(6)];
  p.protocol = PROTOS[g.below(3)];
  p.host_port = PORTS[g.below(7)];
  p.container_port = p.host_port > 0 ? p.host_port : 80;
  return p;
}

static void print_packed(const PackedHostPorts& pk) {
  std::string ents = "[";
  for (size_t k = 0; k < pk.port.size(); ++k)
    ents += (k ? ", " : "") + std::string("[") + std::to_string(pk.ip[k]) + ", " + std::to_string(pk.protocol[k]) +
            ", " + std::to_string(pk.port[k]) + "]";
  printf("\"packed\": {\"entries\": %s], \"used\": %s, \"want\": %s}", ents.c_str(), jnums(pk.used).c_str(),
         jnums(pk.want).c_str());
}

int main(int argc, char** argv) {
  const bool gpu = argc > 1 && !strcmp(argv[1], "gpu");
  const size_t N = 8, P = 20;
  printf("{\"scenarios\": [");
  for (int sc = 0; sc < 3; ++sc) {
    Gen g(4242 + sc);
    std::vector<Node> nodes(N);
    std::vector<NodeInfo> infos(N);
    for (size_t i = 0; i < N; ++i) {
      nodes[i].name = "node-" + std::to_string(i);
      nodes[i].allocatable = {{"cpu", "64"}, {"memory", "256Gi"}, {"pods", "110"}};
      infos[i].node = &nodes[i];
      const uint32_t nu = g.below(3);
      for (uint32_t k = 0; k < nu; ++k) infos[i].used_ports.push_back(random_port(g));
    }
    std::vector<Pod> pods(P);
    for (size_t p = 0; p < P; ++p) {
      pods[p].ns = "default";
      pods[p].name = "p" + std::to_string(p);
      pods[p].uid = "uid-p" + std::to_string(p);
      pods[p].queue_ts_ns = (int64_t)p;
      const uint32_t nc = 1 + g.below(2);
      for (uint32_t c = 0; c < nc; ++c) {
        Container ct;
        ct.requests = {{"cpu", "1"}, {"memory", "1Gi"}};
        const uint32_t np = g.below(3);
        for (uint32_t k = 0; k < np; ++k) ct.ports.push_back(random_port(g));
        pods[p].containers.push_back(ct);
      }
    }
    std::vector<const NodeInfo*> snap;
    for (auto& ni : infos) snap.push_back(&ni);
    std::vector<const Pod*> pend;
    for (auto& p : pods) pend.push_back(&p);

    printf("%s{\"nodes\": [", sc ? ", " : "");
    for (size_t i = 0; i < N; ++i) printf("%s%s", i ? ", " : "", jports(infos[i].used_ports).c_str());
    printf("], \"pods\": [");
    for (size_t p = 0; p < P; ++p) {
      std::vector<ContainerPort> all;
      for (const Container& c : pods[p].containers) all.insert(all.end(), c.ports.begin(), c.ports.end());
      printf("%s%s", p ? ", " : "", jports(all).c_str());
    }
    printf("], ");
    PackedHostPorts pk;
    const Status st = BatchSchedulingPlugin::PackHostPorts(snap, pend, &pk);
    if (!st.ok()) { fprintf(stderr, "%s\n", st.message.c_str()); return 1; }
    print_packed(pk);

    if (gpu && sc == 0) {
      BatchSchedulingPlugin plg(0, 0, BS_OUT_FIT_BITMAP | BS_OUT_REASONS);
      plg.SetHostPortFilter(true);
      const Status rs = plg.BeginRound(snap, pend, 1000000000ll);
      if (!rs.ok()) { fprintf(stderr, "round failed: %s\n", rs.message.c_str()); return 1; }
      auto print_round = [&](const char* key) {
        printf(", \"%s\": [", key);
        for (size_t p = 0; p < P; ++p)
          printf("%s{\"fit_error\": %s, \"reasons\": %s, \"host_ports\": %s}", p ? ", " : "",
                 q(plg.FitError(pods[p].uid)).c_str(), jnums(plg.ReasonCounts(pods[p].uid)).c_str(),
                 jnums(plg.HostPortReasonCounts(pods[p].uid)).c_str());
        printf("]");
      };
      printf(", \"lanes\": %u", plg.packed().lanes);
      print_round("round");
      std::vector<BatchSchedulingPlugin::ReplayDecision> dec;
      std::vector<BatchSchedulingPlugin::Preemption> pre;
      std::string node;
      std::vector<std::string> victims;
      const bool replay = plg.ReplayQueue(&dec).ok();
      const bool r1 = !plg.Preempt(pods[0].uid, &node, &victims).ok(), r2 = !plg.PreemptAll(&pre).ok(),
                 r3 = !plg.PreemptQueue(&pre, false).ok();
      std::vector<int32_t> placed;   // by queue position
      for (const auto& d : dec) placed.push_back(d.node);
      printf(", \"replay_runs\": %s, \"replay_nodes\": %s, \"queue\": %s, \"refused\": [%s, %s, %s]",
             replay ? "true" : "false", jnums(placed).c_str(), jnums(plg.queue_order()).c_str(), r1 ? "true" : "false",
             r2 ? "true" : "false", r3 ? "true" : "false");
      // node 0 takes every port any pod wants: the switch repacks on UpdateNodes and on UpdateRound
      NodeInfo full = infos[0];
      for (const Pod& p : pods)
        for (const Container& c : p.containers) full.used_ports.insert(full.used_ports.end(), c.ports.begin(), c.ports.end());
      const Status us = plg.UpdateNodes({{0u, &full}});
      printf(", \"node0_ports\": %s, \"update_nodes_ok\": %s", jports(full.used_ports).c_str(), us.ok() ? "true" : "false");
      print_round("after_update_nodes");
      const Status ur = plg.UpdateRound({{0u, &infos[0]}}, {}, 3000000000ll);
      printf(", \"update_round_ok\": %s", ur.ok() ? "true" : "false");
      print_round("after_update_round");
    }
    printf("}");
  }
  // 65 distinct wanted entries cannot be packed
  {
    Pod big;
    big.ns = "default";
    big.name = big.uid = "big";
    Container c;
    for (int k = 0; k < 65; ++k) {
      ContainerPort cp;
      cp.host_port = 1000 + k;
      c.ports.push_back(cp);
    }
    big.containers.push_back(c);
    PackedHostPorts pk;
    const Status s65 = BatchSchedulingPlugin::PackHostPorts({}, {&big}, &pk);
    big.containers[0].ports.pop_back();
    const Status s64 = BatchSchedulingPlugin::PackHostPorts({}, {&big}, &pk);
    printf("], \"refuses_65\": %s, \"packs_64\": %s, \"entries_64\": %zu}\n", s65.ok() ? "false" : "true",
           s64.ok() ? "true" : "false", pk.port.size());
  }
  return 0;
}
