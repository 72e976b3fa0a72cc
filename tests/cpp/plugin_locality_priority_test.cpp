// plugin_locality_priority_test.cpp — BatchSchedulingPlugin::PackLocality and SetLocalityWeights, printed as JSON for
// tests/test_plugin_locality_priority.py (CPU) and tests/test_gpu_locality_priority.py (GPU).  One fixed round of five
// nodes (images under several names, one name reported with two sizes, a name that only matches before
// normalization, preferAvoidPods entries of RS, RC and other kinds) and eight pending pods (untagged, tagged and
// registry-port images, a repeated image, two pods with the same images in another order, no containers, controllers
// of every kind).  The program prints the objects themselves, so that the test evaluates them independently, and
// what PackLocality made of them; also whether 64 and 65 avoided controllers pack.  With the argument "gpu" it also
// runs the round on the device with SetLocalityWeights(1, 10000) and prints PriorityNodes and ReplayQueue(kPriority)
// next to the lists and the walk of an engine called directly with the packed tables.
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../batch-scheduler_b200/csrc/plugin.hpp"

using namespace bsched;

static std::string q(const std::string& s) { return "\"" + s + "\""; }
static constexpr int64_t MiB = 1ll << 20;

static int packs(size_t n_controllers) {
  std::vector<Node> nodes(1);
  std::vector<NodeInfo> infos(1);
  std::vector<Pod> pods(n_controllers);
  for (size_t k = 0; k < n_controllers; ++k) {
    nodes[0].prefer_avoid_pods.push_back(PodController{"ReplicaSet", "rs-" + std::to_string(k)});
    pods[k].controller_kind = "ReplicaSet";
    pods[k].controller_uid = "rs-" + std::to_string(k);
  }
  nodes[0].name = "n0";
  infos[0].node = &nodes[0];
  std::vector<const NodeInfo*> snap{&infos[0]};
  std::vector<const Pod*> pend;
  for (auto& p : pods) pend.push_back(&p);
  PackedLocality pl;
  return BatchSchedulingPlugin::PackLocality(snap, pend, &pl).ok() ? (int)pl.controllers.size() : -1;
}

int main(int argc, char** argv) {
  const bool gpu = argc > 1 && !strcmp(argv[1], "gpu");
  const size_t N = 5, P = 8;
  std::vector<Node> nodes(N);
  std::vector<NodeInfo> infos(N);
  nodes[0].images = {{{"nginx:latest", "docker.io/library/nginx:latest"}, 100 * MiB},
                     {{"registry:5000/team/train:v2"}, 5000 * MiB}};
  nodes[0].prefer_avoid_pods = {{"ReplicaSet", "rs-1"}, {"Deployment", "d-1"}};
  nodes[1].images = {{{"nginx:latest"}, 120 * MiB}, {{"cuda:12"}, 8000 * MiB}};
  nodes[1].prefer_avoid_pods = {{"ReplicationController", "rc-1"}};
  nodes[2].images = {{{"registry:5000/team/train"}, 1000 * MiB}, {{"unused:1"}, 1000 * MiB}};
  nodes[2].prefer_avoid_pods = {{"ReplicaSet", "rs-2"}, {"ReplicaSet", "rs-9"}};
  nodes[3].images = {{{"cuda:12", "cuda:latest"}, 8000 * MiB}, {{"registry:5000/team/train:latest"}, 3000 * MiB}};
  nodes[4].prefer_avoid_pods = {{"ReplicaSet", "rs-1"}};
  for (size_t i = 0; i < N; ++i) {
    nodes[i].name = "node-" + std::to_string(i);
    nodes[i].allocatable = {{"cpu", "16"}, {"memory", "64Gi"}, {"pods", "110"}};
    infos[i].node = &nodes[i];
  }
  const std::vector<std::vector<std::string>> images = {
      {"nginx"}, {"nginx", "nginx"}, {"registry:5000/team/train:v2", "cuda:12"}, {"registry:5000/team/train"},
      {"cuda:12", "registry:5000/team/train:v2"}, {"busybox"}, {}, {"cuda"}};
  const std::vector<std::pair<std::string, std::string>> ctrl = {
      {"ReplicaSet", "rs-1"}, {"ReplicationController", "rc-1"}, {"StatefulSet", "ss-1"}, {"ReplicaSet", "rs-2"},
      {"", ""}, {"ReplicaSet", "rs-1"}, {"ReplicaSet", "rs-3"}, {"Deployment", "d-1"}};
  std::vector<Pod> pods(P);
  for (size_t p = 0; p < P; ++p) {
    pods[p].ns = "default"; pods[p].name = "pod-" + std::to_string(p); pods[p].uid = "uid-" + std::to_string(p);
    for (const std::string& im : images[p]) {
      Container c;
      c.requests = {{"cpu", "1"}, {"memory", "1Gi"}};
      c.image = im;
      pods[p].containers.push_back(c);
    }
    pods[p].controller_kind = ctrl[p].first;
    pods[p].controller_uid = ctrl[p].second;
    pods[p].queue_ts_ns = (int64_t)p;
  }
  std::vector<const NodeInfo*> snap;
  for (auto& ni : infos) snap.push_back(&ni);
  std::vector<const Pod*> pend;
  for (auto& p : pods) pend.push_back(&p);

  PackedLocality pl;
  const Status st = BatchSchedulingPlugin::PackLocality(snap, pend, &pl);
  if (!st.ok()) { fprintf(stderr, "%s\n", st.message.c_str()); return 1; }

  printf("{\"nodes\": [");
  for (size_t i = 0; i < N; ++i) {
    printf("%s{\"images\": [", i ? ", " : "");
    for (size_t k = 0; k < nodes[i].images.size(); ++k) {
      printf("%s[[", k ? ", " : "");
      for (size_t m = 0; m < nodes[i].images[k].names.size(); ++m)
        printf("%s%s", m ? ", " : "", q(nodes[i].images[k].names[m]).c_str());
      printf("], %lld]", (long long)nodes[i].images[k].size_bytes);
    }
    printf("], \"avoid\": [");
    for (size_t k = 0; k < nodes[i].prefer_avoid_pods.size(); ++k)
      printf("%s[%s, %s]", k ? ", " : "", q(nodes[i].prefer_avoid_pods[k].kind).c_str(),
             q(nodes[i].prefer_avoid_pods[k].uid).c_str());
    printf("]}");
  }
  printf("], \"pods\": [");
  for (size_t p = 0; p < P; ++p) {
    printf("%s{\"images\": [", p ? ", " : "");
    for (size_t k = 0; k < pods[p].containers.size(); ++k) printf("%s%s", k ? ", " : "", q(pods[p].containers[k].image).c_str());
    printf("], \"controller\": [%s, %s]}", q(pods[p].controller_kind).c_str(), q(pods[p].controller_uid).c_str());
  }
  printf("], \"names\": [");
  for (size_t i = 0; i < pl.names.size(); ++i) printf("%s%s", i ? ", " : "", q(pl.names[i]).c_str());
  printf("], \"image_size\": [");
  for (size_t i = 0; i < pl.image_size.size(); ++i) printf("%s%lld", i ? ", " : "", (long long)pl.image_size[i]);
  printf("], \"image_bits\": [");
  for (size_t i = 0; i < pl.image_bits.size(); ++i) printf("%s%u", i ? ", " : "", pl.image_bits[i]);
  printf("], \"image_class\": [");
  for (size_t p = 0; p < P; ++p) printf("%s%u", p ? ", " : "", pl.image_class[p]);
  printf("], \"class_offset\": [");
  for (size_t c = 0; c < pl.class_offset.size(); ++c) printf("%s%u", c ? ", " : "", pl.class_offset[c]);
  printf("], \"class_images\": [");
  for (size_t k = 0; k < pl.class_images.size(); ++k) printf("%s%u", k ? ", " : "", pl.class_images[k]);
  printf("], \"controllers\": [");
  for (size_t b = 0; b < pl.controllers.size(); ++b)
    printf("%s[%s, %s]", b ? ", " : "", q(pl.controllers[b].kind).c_str(), q(pl.controllers[b].uid).c_str());
  printf("], \"avoid_mask\": [");
  for (size_t i = 0; i < N; ++i) printf("%s%llu", i ? ", " : "", (unsigned long long)pl.avoid_mask[i]);
  printf("], \"avoid_bit\": [");
  for (size_t p = 0; p < P; ++p) printf("%s%u", p ? ", " : "", (unsigned)pl.avoid_bit[p]);
  printf("], \"normalized\": [");
  const char* samples[] = {"nginx", "nginx:1.17", "registry:5000/team/app", "registry:5000/team/app:v2", "a/b:c/d"};
  for (size_t k = 0; k < 5; ++k) printf("%s[%s, %s]", k ? ", " : "", q(samples[k]).c_str(), q(normalized_image_name(samples[k])).c_str());
  printf("], \"packs_64\": %d, \"packs_65\": %d", packs(64), packs(65));

  if (gpu) {
    const uint32_t K = 5;
    BatchSchedulingPlugin plg(0, 0, BS_OUT_FIT_BITMAP, 0, K);
    plg.SetLocalityWeights(1, 10000);
    const Status rs = plg.BeginRound(snap, pend, 1000000000ll);
    if (!rs.ok()) { fprintf(stderr, "round failed: %s\n", rs.message.c_str()); return 1; }
    std::vector<BatchSchedulingPlugin::ReplayDecision> dec;
    const Status rq = plg.ReplayQueue(&dec, BatchSchedulingPlugin::ReplayNodeChoice::kPriority);
    if (!rq.ok()) { fprintf(stderr, "replay failed: %s\n", rq.message.c_str()); return 1; }
    // the same round on an engine called directly with the packed tables
    const PackedSnapshot& ps = plg.packed();
    bs_config cfg{0, ps.lanes, BS_OUT_PRIORITY, K};
    bs_engine* e = nullptr;
    int rc = bs_create(&cfg, &e);
    if (rc) { fprintf(stderr, "bs_create: %d\n", rc); return 1; }
    const bs_node_table nt = ps.node_table();
    const bs_group_table gt = ps.group_table();
    const bs_pod_table pt = ps.pod_table();
    std::vector<int64_t> node_nz, pod_nz;
    BatchSchedulingPlugin::PackNonZero(snap, pend, &node_nz, &pod_nz);
    if ((rc = bs_upload_nodes(e, &nt)) || (rc = bs_upload_groups(e, &gt)) || (rc = bs_upload_pods(e, &pt)) ||
        (rc = bs_upload_node_nonzero(e, N, node_nz.data())) || (rc = bs_upload_pod_nonzero(e, P, pod_nz.data())) ||
        (rc = bs_upload_node_locality(e, N, (uint32_t)pl.names.size(), pl.image_size.data(), pl.image_bits.data(),
                                      pl.avoid_mask.data())) ||
        (rc = bs_upload_pod_locality(e, P, pl.image_class.data(), pl.n_classes(), pl.class_offset.data(),
                                     pl.class_images.data(), pl.avoid_bit.data())) ||
        (rc = bs_set_locality_weights(e, 1, 10000))) {
      fprintf(stderr, "engine setup: %d %s\n", rc, bs_last_error(e));
      return 1;
    }
    bs_results res{};
    if ((rc = bs_evaluate(e, &res))) { fprintf(stderr, "bs_evaluate: %d\n", rc); return 1; }
    const std::vector<uint32_t> order = plg.queue_order();   // the queue ReplayQueue walks
    if (order.size() != P) { fprintf(stderr, "queue_order: %zu entries\n", order.size()); return 1; }
    std::vector<int32_t> en(P * K);
    std::vector<int64_t> es(P * K);
    if ((rc = bs_fetch_priority_rows(e, 0, P, en.data(), es.data()))) { fprintf(stderr, "fetch: %d\n", rc); return 1; }
    std::vector<uint8_t> pf(P), rd(P);
    std::vector<int32_t> nd(P);
    bs_replay_result r{};
    r.prefilter = pf.data(); r.node = nd.data(); r.ready = rd.data();
    if ((rc = bs_replay_priority(e, order.data(), P, &r, nullptr))) { fprintf(stderr, "replay: %d\n", rc); return 1; }
    bs_destroy(e);
    printf(", \"plugin\": [");
    for (size_t p = 0; p < P; ++p) {
      printf("%s[", p ? ", " : "");
      size_t k = 0;
      for (auto& kv : plg.PriorityNodes(pods[p].uid)) printf("%s[%s, %lld]", k++ ? ", " : "", q(kv.first).c_str(), (long long)kv.second);
      printf("]");
    }
    printf("], \"engine\": [");
    for (size_t p = 0; p < P; ++p) {
      printf("%s[", p ? ", " : "");
      for (uint32_t k = 0; k < K && en[p * K + k] >= 0; ++k)
        printf("%s[%s, %lld]", k ? ", " : "", q(nodes[en[p * K + k]].name).c_str(), (long long)es[p * K + k]);
      printf("]");
    }
    printf("], \"plugin_replay\": [");
    for (size_t p = 0; p < P; ++p) printf("%s%d", p ? ", " : "", dec[p].node);
    printf("], \"engine_replay\": [");
    std::vector<int32_t> by_pod(P, -1);
    for (size_t qi = 0; qi < P; ++qi) by_pod[order[qi]] = nd[qi];
    for (size_t p = 0; p < P; ++p) printf("%s%d", p ? ", " : "", by_pod[p]);
    printf("]");
  }
  printf("}\n");
  return 0;
}
