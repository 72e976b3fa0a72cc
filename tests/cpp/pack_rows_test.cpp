// pack_rows_test.cpp — the packer's two row encodings against each other; prints JSON for tests/test_pack_rows.py.
//   pack_rows_random [sets] : every node / group row of a full pack re-encoded by PackNodeRows / PackGroupRows (CPU)
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <random>
#include <string>
#include <vector>

#include "../../batch-scheduler_b200/csrc/plugin.hpp"

using namespace bsched;

// Random object sets: every node and group row of a full Pack, re-encoded by PackNodeRows / PackGroupRows under that
// pack's dictionaries, must come out bit for bit the same — the re-pack of a row the informer touched relies on it.
// Rows the dictionaries cannot encode must ask for a full pack instead; ones they can must not.
static int cmd_pack_rows_random(int sets) {
  static const char* kRes[] = {"cpu", "memory", "ephemeral-storage", "pods", "nvidia.com/gpu", "hugepages-2Mi",
                               "example.com/fpga", "attachable-volumes-ebs", "kubernetes.io/batch", "vendor.io/nic",
                               "requests.vendor.io/x", "widgets"};   // the last two: names Resource.Add ignores
  static const char* kQty[] = {"1", "500m", "2Gi", "1.5", "3k", "100", "0"};
  static const char* kKeys[] = {"zone", "disk", "rack", "gpu"};
  static const char* kVals[] = {"a", "b", "c"};
  static const char* kEffects[] = {"NoSchedule", "NoExecute", "PreferNoSchedule"};
  int bad = 0, nrows = 0, grows = 0, full_rows = 0, triggers = 0, fired = 0, false_full = 0;
  std::map<std::string, int> cover;
  for (int set = 0; set < sets; ++set) {
    std::mt19937_64 rng(4321 + set);
    auto rnd = [&](uint64_t n) { return (uint32_t)(rng() % n); };
    const bool big = set % 8 == 7;   // enough objects for the packer's threads
    const uint32_t N = big ? 2500 : 1 + rnd(150), P = big ? 2000 : rnd(200), G = big ? 500 : 1 + rnd(60);
    auto res_list = [&]() {
      ResourceList rl;
      for (uint32_t k = rnd(6); k > 0; --k) rl.push_back({kRes[rnd(12)], kQty[rnd(7)]});
      return rl;
    };
    auto pick_pod = [&](Pod& p, bool many_pairs, uint32_t i) {
      p.ns = "default"; p.name = "pod-" + std::to_string(i); p.uid = "uid-" + std::to_string(i);
      for (uint32_t k = rnd(3); k > 0; --k) p.node_selector[kKeys[rnd(4)]] = kVals[rnd(3)];
      if (many_pairs && rnd(2)) p.node_selector["k" + std::to_string(i % 80)] = "v";
      for (uint32_t k = rnd(3); k > 0; --k) {
        Toleration t;
        if (rnd(3)) t.key = kKeys[rnd(4)];
        t.op = rnd(3) == 0 ? "Exists" : rnd(2) ? "Equal" : "";
        t.value = rnd(2) ? kVals[rnd(3)] : "";
        if (rnd(2)) t.effect = kEffects[rnd(3)];
        p.tolerations.push_back(t);
      }
      if (rnd(4) == 0) {
        p.has_required_affinity = true;
        for (uint32_t k = rnd(3); k > 0; --k) {
          NodeSelectorTerm t;
          NodeSelectorRequirement r; r.key = kKeys[rnd(4)]; r.op = rnd(2) ? "In" : "NotIn"; r.values = {kVals[rnd(3)]};
          t.match_expressions.push_back(r);
          p.required_affinity.push_back(t);
        }
      }
      for (uint32_t k = 1 + rnd(2); k > 0; --k) {
        Container c; c.has_limits = rnd(2); c.limits = res_list(); c.requests = res_list();
        p.containers.push_back(c);
      }
    };
    std::vector<Node> nodes(N);
    std::vector<NodeInfo> infos(N);
    std::vector<const NodeInfo*> snap(N);
    for (uint32_t i = 0; i < N; ++i) {
      Node& nd = nodes[i];
      nd.name = "node-" + std::to_string(i);
      for (uint32_t k = rnd(4); k > 0; --k) nd.labels[kKeys[rnd(4)]] = kVals[rnd(3)];
      if (set % 2) for (int k = 0; k < 80; ++k) if ((i + k) % 3 == 0) nd.labels["k" + std::to_string(k)] = "v";
      for (uint32_t k = rnd(4); k > 0; --k) nd.taints.push_back({kKeys[rnd(4)], rnd(2) ? kVals[rnd(3)] : "", kEffects[rnd(3)]});
      nd.allocatable = res_list();
      nd.unschedulable = rnd(6) == 0;
      NodeInfo& ni = infos[i];
      ni.node = rnd(12) == 0 ? nullptr : &nd;
      ni.requested = res_list();
      ni.num_pods = (int32_t)rnd(100);
      ni.taints_error = rnd(10) == 0;
      snap[i] = rnd(15) == 0 ? nullptr : &ni;
    }
    // odd sets: more than 64 distinct selector pairs, so every nodeSelector moves into the affinity table
    std::vector<Pod> pods(P), reps(G);
    std::vector<const Pod*> pending(P);
    for (uint32_t i = 0; i < P; ++i) { pick_pod(pods[i], set % 2, i); pending[i] = &pods[i]; }
    std::vector<PodGroup> groups(G);
    std::vector<BatchSchedulingPlugin::GroupDelta> gd(G);
    for (uint32_t g = 0; g < G; ++g) {
      PodGroup& pg = groups[g];
      pg.ns = "default"; pg.name = "pg-" + std::to_string(rnd(G)); pg.min_member = rnd(9); pg.scheduled = rnd(4);
      pg.creation_ns = rnd(1000); pg.max_schedule_time_ns = rnd(2) ? -1 : (int64_t)rnd(100) * 1000000000ll;
      if ((pg.has_min_resources = rnd(2))) pg.min_resources = res_list();
      gd[g].index = g; gd[g].pg = &pg; gd[g].matched = rnd(10); gd[g].flags = (uint8_t)rnd(256);
      const uint32_t r = rnd(3);
      if (r == 1 && P) gd[g].rep_pod = &pods[rnd(P)];
      else if (r == 2) { pick_pod(reps[g], set % 2, P + g); gd[g].rep_pod = &reps[g]; }
    }
    const int64_t wait = 5000000000ll;
    PackedSnapshot full;
    Status st = BatchSchedulingPlugin::Pack(snap, pending, gd, {}, wait, &full);
    if (!st.ok()) { fprintf(stderr, "set %d: pack failed: %s\n", set, st.message.c_str()); return 1; }
    const uint32_t L = full.lanes;
    cover["sel_in_table"] += full.sel_in_table;
    cover["sel_in_masks"] += !full.sel_in_table && !full.sel_pairs.empty();
    cover["aff_classes"] += full.n_aff() > 0;
    cover["lanes_ge_6"] += L >= 6;
    for (uint32_t i = 0; i < N; ++i) {
      cover["nil"] += !snap[i];
      if (!snap[i]) continue;
      cover["no_node"] += !snap[i]->node;
      cover["taints_err"] += snap[i]->taints_error;
      if (!snap[i]->node) continue;
      cover["unschedulable"] += nodes[i].unschedulable;
      for (auto& t : nodes[i].taints) cover[t.effect] += 1;
      for (auto& kv : nodes[i].allocatable) cover["ignored_name"] += kv.first == "widgets" || kv.first == "requests.vendor.io/x";
    }
    for (uint32_t g = 0; g < G; ++g) {
      cover[groups[g].has_min_resources ? "min_res" : "no_min_res"] += 1;
      if (!gd[g].rep_pod) continue;
      cover["rep_sel"] += !gd[g].rep_pod->node_selector.empty();
      cover["rep_tol"] += !gd[g].rep_pod->tolerations.empty();
      cover["rep_aff"] += gd[g].rep_pod->has_required_affinity;
    }

    // every node row
    PackedSnapshot node_rows;
    bool needs_full = true;
    st = BatchSchedulingPlugin::PackNodeRows(full, snap, &node_rows, &needs_full);
    if (!st.ok()) { fprintf(stderr, "set %d: node rows: %s\n", set, st.message.c_str()); return 1; }
    full_rows += needs_full;
    nrows += N;
    const uint32_t W = (N + 31) / 32;
    for (uint32_t i = 0; i < N && !needs_full; ++i) {
      int b = 0;
      for (uint32_t d = 0; d < L; ++d)
        b += node_rows.alloc[(size_t)d * N + i] != full.alloc[(size_t)d * N + i] || node_rows.requested[(size_t)d * N + i] != full.requested[(size_t)d * N + i];
      b += node_rows.pod_count[i] != full.pod_count[i] || node_rows.alloc_present[i] != full.alloc_present[i];
      b += node_rows.req_present[i] != full.req_present[i] || node_rows.label_mask[i] != full.label_mask[i];
      b += node_rows.taint_mask[i] != full.taint_mask[i] || node_rows.node_flags[i] != full.node_flags[i];
      for (uint32_t c = 0; c < full.n_aff(); ++c)
        b += (node_rows.aff_bits[(size_t)c * N + i] != 0) != (((full.aff_bits[(size_t)c * W + i / 32] >> (i % 32)) & 1) != 0);
      if (b) fprintf(stderr, "set %d: node row %u differs\n", set, i);
      bad += b;
    }
    // every group row
    PackedSnapshot group_rows;
    needs_full = true;
    st = BatchSchedulingPlugin::PackGroupRows(full, gd, wait, &group_rows, &needs_full);
    if (!st.ok()) { fprintf(stderr, "set %d: group rows: %s\n", set, st.message.c_str()); return 1; }
    full_rows += needs_full;
    grows += G;
    for (uint32_t g = 0; g < G && !needs_full; ++g) {
      int b = 0;
      for (uint32_t d = 0; d < L; ++d) b += group_rows.min_res[(size_t)d * G + g] != full.min_res[(size_t)d * G + g];
      b += group_rows.min_member[g] != full.min_member[g] || group_rows.scheduled[g] != full.scheduled[g] || group_rows.matched[g] != full.matched[g];
      b += group_rows.group_flags[g] != full.group_flags[g] || group_rows.min_res_present[g] != full.min_res_present[g];
      b += group_rows.rep_sel[g] != full.rep_sel[g] || group_rows.rep_tol[g] != full.rep_tol[g] || group_rows.rep_aff[g] != full.rep_aff[g];
      b += group_rows.creation_ns[g] != full.creation_ns[g] || group_rows.wait_ns[g] != full.wait_ns[g] || group_rows.name_rank[g] != full.name_rank[g];
      if (b) fprintf(stderr, "set %d: group row %u differs\n", set, g);
      bad += b;
    }

    // rows outside the dictionaries: (expected needs_full, outcome)
    PackedSnapshot one;
    auto node_case = [&](bool want, void (*edit)(Node&, NodeInfo&)) {
      Node n2; n2.name = "odd"; n2.allocatable = {{"cpu", "4"}};
      NodeInfo i2; i2.node = &n2; i2.requested = {{"memory", "1Gi"}};
      edit(n2, i2);
      bool nf = !want;
      const Status s = BatchSchedulingPlugin::PackNodeRows(full, {&i2}, &one, &nf);
      ++triggers;
      if (s.ok() && nf == want) ++fired; else if (!want) ++false_full;
    };
    auto group_case = [&](bool want, void (*edit)(PodGroup&, Pod&)) {
      PodGroup g2; g2.ns = "default"; g2.name = "odd";
      Pod rep; rep.ns = "default"; rep.name = "odd";
      edit(g2, rep);
      BatchSchedulingPlugin::GroupDelta d; d.index = 0; d.pg = &g2; d.rep_pod = &rep;
      bool nf = !want;
      const Status s = BatchSchedulingPlugin::PackGroupRows(full, {d}, wait, &one, &nf);
      ++triggers;
      if (s.ok() && nf == want) ++fired; else if (!want) ++false_full;
    };
    node_case(true, [](Node& n, NodeInfo&) { n.taints.push_back({"never-seen", "x", "NoSchedule"}); });
    node_case(true, [](Node& n, NodeInfo&) { n.taints.push_back({"never-seen", "x", "NoExecute"}); });
    node_case(true, [](Node& n, NodeInfo&) { n.allocatable.push_back({"example.org/never-seen", "1"}); });
    node_case(true, [](Node&, NodeInfo& i) { i.requested.push_back({"example.org/never-seen", "1"}); });
    node_case(false, [](Node& n, NodeInfo&) { n.taints.push_back({"never-seen", "x", "PreferNoSchedule"}); });
    node_case(false, [](Node& n, NodeInfo& i) { n.allocatable.push_back({"never-seen", "1"}); i.requested.push_back({"requests.x/y", "1"}); });
    group_case(true, [](PodGroup&, Pod& p) { p.node_selector = {{"never", "seen"}}; });
    group_case(true, [](PodGroup&, Pod& p) {
      p.has_required_affinity = true;
      NodeSelectorTerm t; t.match_expressions = {{"never-seen", "In", {"x"}}}; p.required_affinity = {t};
    });
    group_case(true, [](PodGroup& g, Pod&) { g.has_min_resources = true; g.min_resources = {{"example.org/never-seen", "1"}}; });
    group_case(false, [](PodGroup& g, Pod&) { g.has_min_resources = true; g.min_resources = {{"cpu", "1"}, {"never-seen", "1"}}; });
  }
  printf("{\"sets\": %d, \"node_rows\": %d, \"group_rows\": %d, \"mismatches\": %d, \"needs_full\": %d, "
         "\"triggers\": %d, \"fired\": %d, \"false_full\": %d, \"cover\": {", sets, nrows, grows, bad, full_rows, triggers,
         fired, false_full);
  bool first = true;
  for (auto& kv : cover) { printf("%s\"%s\": %d", first ? "" : ", ", kv.first.c_str(), kv.second); first = false; }
  printf("}}\n");
  return 0;
}

int main(int argc, char** argv) {
  if (argc < 2) return 2;
  if (!strcmp(argv[1], "pack_rows_random")) return cmd_pack_rows_random(argc >= 3 ? atoi(argv[2]) : 40);
  return 2;
}
