// plugin_preempt_pdb_test.cpp — PodDisruptionBudgets in preemption through BatchSchedulingPlugin, as JSON for
// tests/test_plugin_preempt_pdb.py.
//   pack   (CPU) PackBoundPods' BS_BOUND_PDB_VIOLATING classification, with and without budgets
//   cases  (GPU) the hand-built cases 1-4 of tests/pdb_cases.py: Preempt, PreemptAll and bs_preempt on the plugin's
//                engine with the packed table
//   setter (GPU) SetPodDisruptionBudgets takes effect at the next BeginRound and at UpdateNodes
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

static Pod make_pod(const std::string& ns, const std::string& name, const char* cpu, int32_t prio, int64_t start,
                    std::map<std::string, std::string> labels) {
  Pod p;
  p.ns = ns; p.name = name; p.uid = "uid-" + name;
  Container c;
  c.requests = {{"cpu", cpu}};
  p.containers = {c};
  p.priority = prio;
  p.start_ns = start;
  p.labels = std::move(labels);
  return p;
}

static PodDisruptionBudget make_pdb(const std::string& ns, const std::string& name, int32_t allowed,
                                    std::map<std::string, std::string> match_labels,
                                    std::vector<LabelSelectorRequirement> exprs = {}, bool has_selector = true) {
  PodDisruptionBudget b;
  b.ns = ns; b.name = name; b.disruptions_allowed = allowed; b.has_selector = has_selector;
  b.selector.match_labels = std::move(match_labels);
  b.selector.match_expressions = std::move(exprs);
  return b;
}

static void print_flags(const char* key, const PackedBound& b) {
  printf("%s: {", json_str(key).c_str());
  for (uint32_t k = 0; k < b.n; ++k) printf("%s%s: %u", k ? ", " : "", json_str(b.pods[k]->name).c_str(), b.flags[k]);
  printf("}");
}

static int cmd_pack() {
  PackedSnapshot ctx;
  ctx.lanes = 4;
  std::vector<Pod> pods = {
      make_pod("ns", "plain", "1", 0, 0, {{"app", "none"}}),
      make_pod("ns", "other-ns", "1", 0, 0, {{"app", "o"}}),        // the budget selecting it lives in namespace "other"
      make_pod("nl", "no-labels", "1", 0, 0, {}),                  // a pod without labels matches no budget
      make_pod("nl", "labelled", "1", 0, 0, {{"x", "1"}}),         // ... the same budget matches a labelled pod
      make_pod("ns", "nil-sel", "1", 0, 0, {{"app", "nil"}}),
      make_pod("ns", "bad-sel", "1", 0, 0, {{"app", "bad"}}),
      make_pod("ns", "allow-1", "1", 0, 0, {{"app", "a1"}}),
      make_pod("ns", "allow-0", "1", 0, 0, {{"app", "a0"}}),
      make_pod("ns", "allow-neg", "1", 0, 0, {{"app", "an"}}),
      make_pod("ns", "two", "1", 0, 0, {{"app", "two"}}),
      make_pod("ns", "locked", "1", 0, 0, {{"app", "a0"}, {kPodGroupLabel, "run"}}),
  };
  const std::vector<PodDisruptionBudget> pdbs = {
      make_pdb("other", "other", 0, {{"app", "o"}}),
      make_pdb("nl", "not-zzz", 0, {}, {{"zzz", "DoesNotExist", {}}}),
      make_pdb("ns", "nil", 0, {{"app", "nil"}}, {}, false),                         // nil: matches nothing
      make_pdb("ns", "empty", 0, {}),                                                // empty: matches nothing
      make_pdb("ns", "bad-in", 0, {{"app", "bad"}}, {{"k", "In", {}}}),              // In without values
      make_pdb("ns", "bad-op", 0, {{"app", "bad"}}, {{"k", "Matches", {"v"}}}),      // unknown operator
      make_pdb("ns", "bad-exists", 0, {{"app", "bad"}}, {{"k", "Exists", {"v"}}}),   // Exists with values
      make_pdb("ns", "allow-1", 1, {{"app", "a1"}}),
      make_pdb("ns", "allow-0", 0, {}, {{"app", "In", {"a0", "zz"}}}),
      make_pdb("ns", "allow-neg", -1, {{"app", "an"}}),
      make_pdb("ns", "two-ok", 5, {{"app", "two"}}),
      make_pdb("ns", "two-spent", 0, {}, {{"app", "Exists", {}}, {"app", "NotIn", {"none", "o", "nil", "bad", "a1", "a0", "an"}}}),
  };
  NodeInfo n0;
  for (const Pod& p : pods) n0.pods.push_back(&p);
  const std::unordered_map<std::string, uint32_t> rows = {{"ns/run", 0}};
  const std::vector<uint8_t> locked = {1};
  PackedBound with, without;
  const Status a = BatchSchedulingPlugin::PackBoundPods(ctx, {&n0}, rows, locked, &with, pdbs);
  const Status b = BatchSchedulingPlugin::PackBoundPods(ctx, {&n0}, rows, locked, &without);
  printf("{\"ok\": %s, ", a.ok() && b.ok() ? "true" : "false");
  print_flags("with", with);
  printf(", ");
  print_flags("without", without);
  printf("}\n");
  return 0;
}

// One scenario on its own plugin: nodes with 2 or 4 cpus fully requested, their bound pods, one pending preemptor
// (priority 100, online) and the budgets.  Bound pods labelled pdb=spent violate the budget "spent".
struct Scenario {
  std::vector<Node> nodes;
  std::vector<NodeInfo> infos;
  std::vector<Pod> bound;
  std::vector<uint32_t> bound_node;
  Pod preemptor;
  void node(const char* cpu) {
    Node n;
    n.name = "node-" + std::to_string(nodes.size());
    n.allocatable = {{"cpu", cpu}, {"memory", "8Gi"}, {"pods", "110"}};
    nodes.push_back(n);
  }
  void pod(uint32_t node, const char* name, const char* cpu, int32_t prio, int64_t start, bool vio) {
    bound.push_back(make_pod("ns", name, cpu, prio, start, vio ? std::map<std::string, std::string>{{"pdb", "spent"}}
                                                               : std::map<std::string, std::string>{{"pdb", "free"}}));
    bound_node.push_back(node);
  }
  std::vector<const NodeInfo*> snapshot() {
    infos.assign(nodes.size(), NodeInfo());
    for (size_t i = 0; i < nodes.size(); ++i) {
      infos[i].node = &nodes[i];
      infos[i].requested = {{"cpu", nodes[i].allocatable[0].second}};
    }
    for (size_t k = 0; k < bound.size(); ++k) infos[bound_node[k]].pods.push_back(&bound[k]);
    std::vector<const NodeInfo*> snap;
    for (auto& ni : infos) {
      ni.num_pods = (int32_t)ni.pods.size();
      snap.push_back(&ni);
    }
    return snap;
  }
};

static std::vector<PodDisruptionBudget> spent_budget() { return {make_pdb("ns", "spent", 0, {{"pdb", "spent"}})}; }

static void print_answer(const std::string& node, const std::vector<std::string>& victims) {
  printf("[%s, [", json_str(node).c_str());
  for (size_t k = 0; k < victims.size(); ++k) printf("%s%s", k ? ", " : "", json_str(victims[k]).c_str());
  printf("]]");
}

static void print_preempt(BatchSchedulingPlugin& plugin, const Pod& p) {
  std::string node;
  std::vector<std::string> victims;
  const Status st = plugin.Preempt(p.uid, &node, &victims);
  print_answer(st.ok() ? node : "error: " + st.message, victims);
}

// bs_preempt on the plugin's engine with the plugin's packed table, for pending row 0
static void print_direct(BatchSchedulingPlugin& plugin, const Scenario& sc) {
  const PackedBound& b = plugin.bound();
  const bs_bound_table t = b.table();
  int rc = bs_upload_bound_pods(plugin.engine(), &t);
  uint32_t row = 0, nv = 0, cand = 0, off[2] = {0, 0};
  int32_t node = -1;
  std::vector<uint32_t> vict(b.n + 1);
  bs_preempt_result r{&node, &nv, &cand, off, vict.data(), (uint32_t)vict.size(), 0};
  if (!rc) rc = bs_preempt(plugin.engine(), &row, 1, &r);
  std::vector<std::string> victims;
  for (uint32_t k = 0; !rc && k < nv; ++k) victims.push_back(b.pods[vict[k]]->uid);
  print_answer(rc ? "error" : node >= 0 ? sc.nodes[node].name : "", victims);
}

static Scenario make_case(int c) {
  Scenario sc;
  sc.preemptor = make_pod("ns", "preemptor", "2", 100, 0, {});
  switch (c) {
    case 1:   // reprieve order: A (10, violating) stays, B (20) goes
      sc.node("4");
      sc.pod(0, "a", "2", 10, 0, true);
      sc.pod(0, "b", "2", 20, 0, false);
      break;
    case 2:   // fewest violations beats the lower priority
      sc.node("2"); sc.node("2");
      sc.pod(0, "v", "2", 0, 0, true);
      sc.pod(1, "w", "2", 50, 0, false);
      break;
    case 3:   // victims[0]'s priority decides: node-0's V (0) before node-1's X (10)
      sc.node("2"); sc.node("2");
      sc.pod(0, "v", "1", 0, 0, true);
      sc.pod(0, "w", "1", 40, 0, false);
      sc.pod(1, "x", "2", 10, 0, true);
      break;
    default:   // 4: the earliest start among the priority-40 victims, the later one wins
      sc.node("2"); sc.node("2");
      sc.pod(0, "v0", "1", 0, 5, true);
      sc.pod(0, "w0", "1", 40, 1, false);
      sc.pod(1, "v1", "1", 0, 1, true);
      sc.pod(1, "w1", "1", 40, 5, false);
      break;
  }
  return sc;
}

static int cmd_cases() {
  printf("{");
  for (int c = 1; c <= 4; ++c) {
    Scenario sc = make_case(c);
    BatchSchedulingPlugin plugin(0, 0, BS_OUT_FIT_BITMAP);
    plugin.SetPodDisruptionBudgets(spent_budget());
    const std::vector<const NodeInfo*> snap = sc.snapshot();
    Status st = plugin.BeginRound(snap, {&sc.preemptor}, 1000000000ll);
    if (!st.ok()) { fprintf(stderr, "round failed: %s\n", st.message.c_str()); return 1; }
    printf("%s\"%d\": {\"preempt\": ", c > 1 ? ", " : "", c);
    print_preempt(plugin, sc.preemptor);
    std::vector<BatchSchedulingPlugin::Preemption> all;
    st = plugin.PreemptAll(&all);
    printf(", \"all\": ");
    if (st.ok() && all.size() == 1 && all[0].uid == sc.preemptor.uid) print_answer(all[0].node, all[0].victims);
    else printf("\"error\"");
    printf(", \"direct\": ");
    print_direct(plugin, sc);
    printf("}");
  }
  printf("}\n");
  return 0;
}

static int cmd_setter() {
  Scenario sc = make_case(2);
  BatchSchedulingPlugin plugin(0, 0, BS_OUT_FIT_BITMAP);
  const std::vector<const NodeInfo*> snap = sc.snapshot();
  Status st = plugin.BeginRound(snap, {&sc.preemptor}, 1000000000ll);
  if (!st.ok()) { fprintf(stderr, "round failed: %s\n", st.message.c_str()); return 1; }
  printf("{\"none\": ");
  print_preempt(plugin, sc.preemptor);
  plugin.SetPodDisruptionBudgets(spent_budget());   // not read until the table is packed again
  printf(", \"set\": ");
  print_preempt(plugin, sc.preemptor);
  st = plugin.UpdateNodes({{0u, snap[0]}});
  if (!st.ok()) { fprintf(stderr, "update failed: %s\n", st.message.c_str()); return 1; }
  printf(", \"update_nodes\": ");
  print_preempt(plugin, sc.preemptor);
  plugin.SetPodDisruptionBudgets({});
  st = plugin.BeginRound(snap, {&sc.preemptor}, 2000000000ll);
  if (!st.ok()) { fprintf(stderr, "round failed: %s\n", st.message.c_str()); return 1; }
  printf(", \"cleared_begin_round\": ");
  print_preempt(plugin, sc.preemptor);
  plugin.SetPodDisruptionBudgets(spent_budget());
  st = plugin.BeginRound(snap, {&sc.preemptor}, 3000000000ll);
  if (!st.ok()) { fprintf(stderr, "round failed: %s\n", st.message.c_str()); return 1; }
  printf(", \"set_begin_round\": ");
  print_preempt(plugin, sc.preemptor);
  printf("}\n");
  return 0;
}

int main(int argc, char** argv) {
  if (argc >= 2 && !strcmp(argv[1], "pack")) return cmd_pack();
  if (argc >= 2 && !strcmp(argv[1], "cases")) return cmd_cases();
  if (argc >= 2 && !strcmp(argv[1], "setter")) return cmd_setter();
  fprintf(stderr, "usage: %s pack|cases|setter\n", argv[0]);
  return 2;
}
