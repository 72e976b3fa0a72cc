// engine.cu — C ABI (include/bsched.h) of the H100 gang-scheduling feasibility engine.
//
// Host side: table validation + upload, class de-duplication of the pre-encoded
// selector/toleration masks, kernel sequencing on one CUDA stream (the queue sort
// runs concurrently on a second stream), result fetch, and the per-call mirrors of
// batchSchedulingPlugin.PreFilter / Permit / Less (batchscheduler.go:102,165,214).
// There is no CPU implementation of the path here: no device -> BS_E_NODEVICE.
#include <cuda_runtime.h>

#include <omp.h>

#include <algorithm>
#include <array>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <thread>
#include <unordered_map>
#include <chrono>
#include <sched.h>
#include <vector>

#include "devmem.hpp"
#include "kernels.cuh"
#include "interpod_filter.cuh"
#include "fit.cuh"
#include "gang_state.hpp"
#include "sort.cuh"
#include "replay.cuh"
#include "preempt.cuh"
#include "priority.cuh"

using namespace bsk;

namespace {

struct DeviceAlloc {
  static cudaError_t alloc(void** p, size_t bytes) { return cudaMalloc(p, bytes); }
  static void free(void* p) { cudaFree(p); }
};
struct PinnedAlloc {
  static cudaError_t alloc(void** p, size_t bytes) { return cudaHostAlloc(p, bytes, cudaHostAllocDefault); }
  static void free(void* p) { cudaFreeHost(p); }
};
// Compressible device memory (devmem.hpp) where the device supports it and the driver grants it, cudaMalloc
// otherwise.  For the score matrix: every element is INT64_MIN or, on a shape with a narrow lane, a score below 2^27,
// so at least half its bytes are zero and the L2 sends it to DRAM in fewer bytes (DESIGN §4).
struct CompressibleAlloc {
  CompMem m;
  int supported = 0;   // CU_DEVICE_ATTRIBUTE_GENERIC_COMPRESSION_SUPPORTED at the last allocation
  cudaError_t alloc(void** p, size_t bytes) {
    supported = compmem_supported();
    if (compmem_alloc(&m, bytes)) {
      *p = m.p;
      return cudaSuccess;
    }
    return cudaMalloc(p, bytes);
  }
  void free(void* p) {
    if (m.p) compmem_free(&m);
    else cudaFree(p);
  }
  bool compressed() const { return m.p != nullptr; }
};

// A block of device or pinned host memory that frees itself.  ensure() only grows it (at least 256 bytes)
// and does not keep the contents when it does.
template <class A>
struct Buf {
  void* p = nullptr;
  size_t cap = 0;
  A a;   // the allocator: what it needs to free the block, and what it reports about it
  Buf() = default;
  Buf(Buf&& o) noexcept { std::swap(p, o.p); std::swap(cap, o.cap); std::swap(a, o.a); }
  Buf& operator=(Buf&& o) noexcept { std::swap(p, o.p); std::swap(cap, o.cap); std::swap(a, o.a); return *this; }
  ~Buf() { reset(); }
  void reset() {
    if (p) a.free(p);
    p = nullptr;
    cap = 0;
  }
  cudaError_t ensure(size_t bytes) {
    if (bytes <= cap) return cudaSuccess;
    reset();
    const size_t want = std::max<size_t>(bytes, 256);
    cudaError_t e = a.alloc(&p, want);
    if (e == cudaSuccess) cap = want;
    else p = nullptr;
    return e;
  }
  template <class T>
  T* as() const { return reinterpret_cast<T*>(p); }
};
using DevBuf = Buf<DeviceAlloc>;
using PinBuf = Buf<PinnedAlloc>;
using ScoreBuf = Buf<CompressibleAlloc>;

// A field of an arena (carve): it neither allocates nor frees.
struct View {
  void* p = nullptr;
  size_t bytes = 0;
  template <class T>
  T* as() const { return reinterpret_cast<T*>(p); }
};

struct Field {
  View* v;
  size_t bytes;
  View* mirror = nullptr;   // the same field in the mirror arena
};

// Lays the fields out back to back in `arena`, each at a 256-byte aligned offset, and points every view
// at its field.  With a `mirror`, the same layout is carved into it for the mirror views.  An arena that
// has to grow loses its contents.  *used gets the bytes the layout takes.
template <size_t K>
cudaError_t carve(DevBuf& arena, const Field (&fields)[K], PinBuf* mirror = nullptr, size_t* used = nullptr) {
  size_t total = 0;
  for (const Field& f : fields) total += (f.bytes + 255) & ~(size_t)255;
  cudaError_t er = arena.ensure(total);
  if (er == cudaSuccess && mirror) er = mirror->ensure(total);
  if (er != cudaSuccess) return er;
  size_t off = 0;
  for (const Field& f : fields) {
    *f.v = View{arena.as<char>() + off, f.bytes};
    if (mirror) *f.mirror = View{mirror->as<char>() + off, f.bytes};
    off += (f.bytes + 255) & ~(size_t)255;
  }
  if (used) *used = total;
  return cudaSuccess;
}

// A CUDA stream or event that is destroyed with its owner; it converts to the handle the runtime takes.
template <class H, cudaError_t (*destroy)(H)>
struct Handle {
  H h = nullptr;
  Handle() = default;
  Handle(const Handle&) = delete;
  Handle& operator=(const Handle&) = delete;
  ~Handle() {
    if (h) destroy(h);
  }
  operator H() const { return h; }
};
using Stream = Handle<cudaStream_t, cudaStreamDestroy>;
using Event = Handle<cudaEvent_t, cudaEventDestroy>;

// a resizable array in pinned host memory: what is DMA'd every round must not be staged through
// pageable memory
template <class T>
struct PinVec {
  PinBuf buf;
  size_t n = 0;
  bool resize(size_t count) {
    if (buf.ensure(std::max<size_t>(count, 1) * sizeof(T)) != cudaSuccess) return false;
    n = count;
    return true;
  }
  T* data() const { return buf.as<T>(); }
  T& operator[](size_t i) const { return buf.as<T>()[i]; }
  size_t size() const { return n; }
};

// (sel, tol, non-zero scalar request mask): the pre-encoded predicates a pod class shares
struct ClassKey {
  uint64_t sel, tol;
  uint32_t nz;
  uint32_t aff;   // affinity class (row of the bs_upload_affinity table) or BS_AFF_NONE
  uint32_t ipf = BS_IPF_NONE;   // MatchInterPodAffinity filter class while the filter is on, else BS_IPF_NONE
  uint64_t hp = 0;              // PodFitsHostPorts conflict mask while the filter is on, else 0
  bool operator==(const ClassKey& o) const {
    return sel == o.sel && tol == o.tol && nz == o.nz && aff == o.aff && ipf == o.ipf && hp == o.hp;
  }
};

// flat open-addressing index ClassKey -> dense id (insertion order)
struct ClassIndex {
  std::vector<ClassKey> keys;
  std::vector<uint32_t> slots;  // id + 1, 0 = empty
  uint32_t mask = 0;
  ClassKey last_key{0, 0, 0xffffffffu, 0};
  uint32_t last_id = 0;
  static uint64_t hash(const ClassKey& k) {
    uint64_t h = k.sel * 0x9E3779B97F4A7C15ull ^ (k.tol + 0x7F4A7C15ull) * 0xBF58476D1CE4E5B9ull ^
                 ((uint64_t)k.nz | ((uint64_t)k.aff << 32)) * 0x94D049BB133111EBull ^ (uint64_t)(k.ipf + 1u) * 0xD6E8FEB86659FD93ull ^
                 k.hp * 0xC2B2AE3D27D4EB4Full;
    return h ^ (h >> 29);
  }
  void clear() {
    keys.clear();
    slots.assign(256, 0);
    mask = 255;
    last_key = ClassKey{0, 0, 0xffffffffu, 0};
  }
  void grow() {
    std::vector<uint32_t> ns((size_t)(mask + 1) * 2, 0);
    const uint32_t nm = (uint32_t)ns.size() - 1;
    for (uint32_t id = 0; id < keys.size(); ++id) {
      uint32_t s = (uint32_t)hash(keys[id]) & nm;
      while (ns[s]) s = (s + 1) & nm;
      ns[s] = id + 1;
    }
    slots.swap(ns);
    mask = nm;
  }
  uint32_t get_or_add(const ClassKey& k) {
    if (k == last_key) return last_id;
    if (slots.empty()) clear();
    uint32_t s = (uint32_t)hash(k) & mask;
    while (slots[s]) {
      if (keys[slots[s] - 1] == k) {
        last_key = k;
        last_id = slots[s] - 1;
        return last_id;
      }
      s = (s + 1) & mask;
    }
    const uint32_t id = (uint32_t)keys.size();
    keys.push_back(k);
    slots[s] = id + 1;
    if (keys.size() * 2 > slots.size()) grow();
    last_key = k;
    last_id = id;
    return id;
  }
  size_t size() const { return keys.size(); }
};

// Threads for the host packing passes.  Not taken from OMP_NUM_THREADS (launchers such as torchrun
// pin it to 1): BS_HOST_THREADS if set, else the cores divided by the GPUs of the box, at most 8.
inline int host_threads() {
  static int n = [] {
    if (const char* s = getenv("BS_HOST_THREADS")) return std::max(1, atoi(s));
    int ndev = 1;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev < 1) ndev = 1;
    int hw = (int)std::thread::hardware_concurrency();
    cpu_set_t set;   // cores this process may actually run on (cgroup / taskset), not the box's total
    if (sched_getaffinity(0, sizeof(set), &set) == 0 && CPU_COUNT(&set) > 0) hw = std::min(hw > 0 ? hw : 1 << 20, CPU_COUNT(&set));
    return std::max(1, std::min(8, hw / ndev));
  }();
  return n;
}

// The rows [0, n) of a host pass cut into T fixed chunks: one chunk below `serial_below` rows, else host_threads().
// T fixed CHUNKS, not T threads: num_threads(T) is only a request (OMP_THREAD_LIMIT, OMP_DYNAMIC, a failed thread
// creation give a smaller team), so the chunks are shared out with an omp for and a smaller team still covers them.
struct Chunks {
  uint32_t n;
  int T;
  Chunks(uint32_t n_, uint32_t serial_below) : n(n_), T(n_ < serial_below ? 1 : host_threads()) {}
  // body(chunk, first row, end row) for every chunk
  template <class F>
  void run(F body) const {
    const uint32_t chunk = (n + T - 1) / T;
#pragma omp parallel for schedule(static, 1) num_threads(T) if (T > 1)
    for (int t = 0; t < T; ++t) {
      const uint32_t a = std::min(n, (uint32_t)t * chunk);
      body(t, a, std::min(n, a + chunk));
    }
  }
  // body(chunk, first row, end row, the chunk's statistics) for every chunk; returns the chunks' statistics merged
  template <class S, class F>
  S reduce(F body) const {
    std::vector<S> part(T);
    run([&](int t, uint32_t a, uint32_t b) { body(t, a, b, part[t]); });
    S r;
    for (const S& s : part) r.merge(s);
    return r;
  }
};

// What the node pass (node_host_pass) gathers: |value| maxima of alloc / requested (range check + lane classification,
// wide / narrow), max |pod_count|, and per lane the OR and max |value| of the residual at percent 1.0
// (singleNodeResource, core.go:647-668; the OR's trailing zeros are the power of two every residual is a multiple of:
// scaled lanes).  A row update only widens them (a conservative bound keeps the lane split exact; more OR bits give a
// smaller unit, still exact).
struct NodeStats {
  int64_t max_alloc[BS_MAX_LANES] = {}, max_requested[BS_MAX_LANES] = {}, max_left[BS_MAX_LANES] = {};
  uint64_t or_left[BS_MAX_LANES] = {};
  int64_t max_pod_count = 0;
  bool bad_range = false;   // an alloc / requested value outside +-2^56
  void merge(const NodeStats& o) {
    for (uint32_t d = 0; d < BS_MAX_LANES; ++d) {
      max_alloc[d] = std::max(max_alloc[d], o.max_alloc[d]);
      max_requested[d] = std::max(max_requested[d], o.max_requested[d]);
      max_left[d] = std::max(max_left[d], o.max_left[d]);
      or_left[d] |= o.or_left[d];
    }
    max_pod_count = std::max(max_pod_count, o.max_pod_count);
    bad_range = bad_range || o.bad_range;
  }
};

// What the group pass (group_host_pass) gathers: the OR / AND of the two sort-key words (creation_ns, ~name_rank) and
// the checks.  A row update widens the OR / AND: a superset of the varying bits costs a radix pass, never an error.
struct GroupStats {
  uint64_t or_creation = 0, and_creation = ~0ull, or_name = 0, and_name = ~0ull;
  bool bad_range = false;      // a min_res value outside +-2^56
  bool bad_creation = false;   // creation_ns == INT64_MAX
  bool reps_differ = false;    // the representative columns differ from the engine's
  void merge(const GroupStats& o) {
    or_creation |= o.or_creation; and_creation &= o.and_creation;
    or_name |= o.or_name; and_name &= o.and_name;
    bad_range = bad_range || o.bad_range;
    bad_creation = bad_creation || o.bad_creation;
    reps_differ = reps_differ || o.reps_differ;
  }
  // bits that differ between rows of each sort-key word (a constant byte needs no radix pass); AND is a subset of OR
  // once a row was seen, so OR & ~AND is OR ^ AND there and 0 for an empty table
  uint64_t vary_creation() const { return or_creation & ~and_creation; }
  uint64_t vary_name() const { return or_name & ~and_name; }
};

// What the pod pass gathers: per lane max |req| and the largest negative request (0 when none; the replay's
// overflow bound), the OR of every request (scaled lanes), the OR / AND of the sort-key columns, whether a pod sorts
// as ungrouped (lister miss or gid < BS_GID_NONE) and the largest gid.
struct PodStats {
  int64_t max_req[BS_MAX_LANES] = {}, neg_req[BS_MAX_LANES] = {};
  uint64_t or_req[BS_MAX_LANES] = {};
  uint64_t or_ts = 0, and_ts = ~0ull;
  uint32_t or_prio = 0, and_prio = ~0u;
  bool lister_miss = false;
  int32_t max_gid = -1;
  bool bad_range = false;   // a request outside +-2^56
  void merge(const PodStats& o) {
    for (uint32_t d = 0; d < BS_MAX_LANES; ++d) {
      max_req[d] = std::max(max_req[d], o.max_req[d]);
      neg_req[d] = std::max(neg_req[d], o.neg_req[d]);
      or_req[d] |= o.or_req[d];
    }
    or_ts |= o.or_ts; and_ts &= o.and_ts;
    or_prio |= o.or_prio; and_prio &= o.and_prio;
    lister_miss = lister_miss || o.lister_miss;
    max_gid = std::max(max_gid, o.max_gid);
    bad_range = bad_range || o.bad_range;
  }
  uint64_t vary_ts() const { return or_ts & ~and_ts; }   // as GroupStats::vary_creation
  uint64_t vary_prio() const { return or_prio & ~and_prio; }
};

// Merges the chunks' thread-local class indices into `global` (ids of known classes are stable: the index only
// grows), then rewrites every ids[i], an id in the local index of row i's chunk, as its id in `global`.
void merge_classes(ClassIndex& global, const std::vector<ClassIndex>& local, const Chunks& ch, uint32_t* ids) {
  std::vector<std::vector<uint32_t>> remap(local.size());
  for (size_t t = 0; t < local.size(); ++t) {
    remap[t].resize(local[t].size());
    for (size_t j = 0; j < local[t].size(); ++j) remap[t][j] = global.get_or_add(local[t].keys[j]);
  }
  ch.run([&](int t, uint32_t a, uint32_t b) {
    const uint32_t* rm = remap[t].data();
    for (uint32_t i = a; i < b; ++i) ids[i] = rm[ids[i]];
  });
}

// out[i] = id of key_of(i) in `global`: thread-local indices in parallel, then merge_classes.
template <class KeyFn>
void assign_classes(ClassIndex& global, uint32_t n, KeyFn key_of, uint32_t* out) {
  if (global.slots.empty()) global.clear();
  const Chunks ch(n, 8192);
  std::vector<ClassIndex> local(ch.T);
  ch.run([&](int t, uint32_t a, uint32_t b) {
    ClassIndex& li = local[t];
    li.clear();
    for (uint32_t i = a; i < b; ++i) out[i] = li.get_or_add(key_of(i));
  });
  merge_classes(global, local, ch, out);
}

// The node side of InterPodAffinity and of the MatchInterPodAffinity filter (bs_interpod_nodes): topology values
// [keys][N], each term's key and first (term, value) slot, the bound pods and their class table.
struct InterpodNodeSide {
  DevBuf d_topo, d_term_key, d_term_off, d_bound_node, d_bound_class, d_boff, d_bterm, d_bown, d_bmatch;
  uint32_t terms = 0, bound = 0, bclasses = 0;
  uint64_t slots = 0;
};

}  // namespace

struct bs_engine {
  std::mutex mu;
  int device = 0;
  uint32_t L = 0, out_flags = 0;
  uint32_t topk = 0;   // list length K of BS_OUT_TOPK, 0 without it
  Stream s, s2, s3, s4;   // main; queue sort; PreFilter chain (high priority); peer wait
  Event ev_fork, ev_join, ev_pre, ev_push, ev_gath;
  std::string err;
  uint64_t launches = 0;

  // shapes
  uint32_t N = 0, Npad = 0, W = 0, P = 0, G = 0;
  bool have_nodes = false, have_pods = false, have_groups = false;
  bool nodes_dirty = true, classes_dirty = true, evaluated = false;

  // node table (device, padded to Npad) + derived
  DevBuf d_alloc, d_requested, d_pod_count, d_apres, d_rpres, d_label, d_taint, d_nflags;
  DevBuf d_left_w, d_left_n, d_left_present, d_classfit, d_left_plain, d_filter_bitmap;
  LaneMap lane_map{};
  bool lane_map_valid = false;
  // statistics of the tables as uploaded, widened by row updates (lane classification, sort passes, replay bound)
  NodeStats node_stats;
  GroupStats group_stats;
  PodStats pod_stats;
  uint32_t score_pitch = 0;             // elements per score row: N rounded up to even
  uint32_t bitmap_pitch = 0;            // words per fit-bitmap row: ceil(N/32) rounded up to 32 (whole 128-byte lines)
  // pod table
  DevBuf d_req, d_ppres, d_gid, d_prio, d_ts, d_pflags, d_pod_fit_class, d_pod_rep_class;
  // group table
  DevBuf d_min_member, d_scheduled, d_matched, d_gflags, d_min_res, d_mrpres, d_creation, d_name_rank,
      d_group_rep_class;
  // class tables
  DevBuf d_fsel, d_ftol, d_fnz, d_faff, d_rsel, d_rtol, d_raff;
  // affinity bit table (bs_upload_affinity): [n_aff][W] host-evaluated node predicates
  DevBuf d_aff_bits;
  uint32_t n_aff = 0;
  std::vector<uint32_t> h_gaff;   // affinity class of each group's representative pod
  // gang state (SURVEY 8(f) row 3): the reference's TTL tables around Permit, see gang_state.hpp
  GangState gang;
  std::vector<uint32_t> h_min_member, h_scheduled, h_matched_up;   // group columns as uploaded
  std::vector<uint8_t> h_gflags_up;
  std::vector<uint64_t> h_pod_uid, h_pod_name;                     // bs_set_pod_ids
  int64_t cycle_now_ns = 0;
  bool gang_applied = false;     // the round's new_denied have been added to the deny table
  uint32_t n_fit_classes = 0, n_rep_classes = 0;
  // effective group state + round scratch
  DevBuf d_eflags, d_emin_res, d_emrpres, d_erep_class, d_first_pod, d_in_round, d_contrib, d_done, d_okA;
  DevBuf d_pre, d_pre_present, d_pre_stats, d_max_partial, d_pre_part, d_pre_part_pres, d_pre_cstats;
  DevBuf d_pre_done;   // kept between rounds: zeroed only when it is allocated
  uint32_t prefix_slots = 0;
  // outputs
  DevBuf d_stage;         // bs_update_nodes / bs_update_groups: device staging of the changed rows
  DevBuf d_best_packed;   // gang_fit tail pieces: max((score + 1) << 32 | ~node) per pod
  DevBuf d_fit_bitmap;
  ScoreBuf d_score;   // compressible where granted (bs_score_memory); the fit bitmap gains nothing from it
  DevBuf d_topk_node, d_topk_score;   // BS_OUT_TOPK: [Prows][topk] lists
  // BS_OUT_REASONS: full-width residuals [L][Npad], per fit class the gate bitmap [classes][Npad/32] and bins 0-3
  // [classes][4] (rebuilt with the class fit bits), and the rows [P][4 + L]
  DevBuf d_left_full, d_reason_gate, d_reason_class, d_reasons;
  // BS_OUT_PRIORITY: the non-zero request columns (node [2][Npad] zero-padded, pod [2][P]; each dropped with its
  // table), the score weights, and the lists [P][topk]; the fit set is the reason rows' (d_left_full, d_reason_gate)
  DevBuf d_prio_node, d_prio_score;
  struct {
    DevBuf d_node, d_pod;
    bool have_node = false, have_pod = false;
    int64_t node_max[2] = {0, 0}, pod_max[2] = {0, 0};   // per row, of the uploaded columns (bs_replay_priority)
  } nz;
  ScoreWeights weights{1, 0, 1};
  // RequestedToCapacityRatio (bs_set_ratio_priority): weight 0 = off; the shape table lives in d_ratio_tab
  RatioSetting ratio{};
  DevBuf d_ratio_tab;
  // TaintToleration and preferred NodeAffinity (bs_set_node_priority_weights; 0, 0 = off): the node side
  // (PreferNoSchedule masks [Npad], the class x node weights [classes][Npad]; dropped with the node table) and the pod
  // side (tolerated masks [P], the class of each pod [P]; dropped with the pod table).  class_max: the largest class a
  // pod names (-1 none), checked against classes at evaluation.
  uint32_t w_taint = 0, w_naff = 0;
  struct {
    DevBuf d_prefer_taints, d_weights, d_prefer_tol, d_class;
    bool have_node = false, have_pod = false;
    uint32_t classes = 0;
    int64_t class_max = -1;
  } pref;
  // ImageLocality and NodePreferAvoidPods (bs_set_locality_weights; 0, 0 = off): the node side (the image bit rows
  // [n_images][ceil(N/32)] and sizes, the preferAvoidPods masks [Npad]; dropped with the node table) and the pod side
  // (each pod's image class [P], the classes' CSR, each pod's controller bit [P]; dropped with the pod table); each
  // side has its image part and its avoid part.  d_img_scaled and the class x node IL table d_il are built on the
  // device when dirty (priority.cuh image_spread_kernel, locality_class_kernel).  class_max / image_max: the largest
  // class a pod names and the largest id a class lists (-1 none), checked at evaluation.
  uint32_t w_img = 0, w_avoid = 0;
  struct {
    DevBuf d_img_bits, d_img_size, d_img_scaled, d_avoid_mask, d_class, d_off, d_ids, d_avoid_bit, d_il;
    bool have_img_node = false, have_avoid_node = false, have_img_pod = false, have_avoid_pod = false;
    bool dirty = true;
    uint32_t images = 0, classes = 0;
    int64_t class_max = -1, image_max = -1;
  } loc;
  // SelectorSpread (bs_set_spread_weight; 0 = off): the node side (each node's zone [Npad], the class x node counts
  // [classes][Npad]; dropped with the node table) and the pod side (each pod's class [P]; dropped with the pod table).
  // class_max: the largest class a pod names (-1 none), checked against classes at evaluation.
  uint32_t w_spread = 0;
  struct {
    DevBuf d_zone, d_counts, d_class;
    bool have_node = false, have_pod = false;
    uint32_t classes = 0;
    int64_t class_max = -1;
  } spread;
  // InterPodAffinity (bs_set_interpod_weight; 0 = off): the node side (InterpodNodeSide; dropped with the node table)
  // and the pod side (each pod's class [P] and the class table; dropped with the pod table).  d_ms (M and S per slot)
  // and the pod class x node raw table d_raw are built on the device when dirty (mass_dirty: M and S too).
  // term_max: the largest term a pod class names (-1 none), checked against node.terms at evaluation.
  uint32_t w_ipa = 0;
  struct {
    InterpodNodeSide node;
    DevBuf d_ms, d_class, d_poff, d_pterm, d_pown, d_pmatch, d_raw;
    bool have_node = false, have_pod = false, dirty = true, mass_dirty = true;
    uint32_t pclasses = 0;
    int64_t term_max = -1;
  } ipa;
  // MatchInterPodAffinity filter (bs_set_interpod_filter; off by default): the node side (InterpodNodeSide; dropped
  // with the node table) and the pod side (each pod's filter class h_class, the class table; dropped with the pod
  // table).  The presence planes d_presence ([2][words]: match, own), the per-term counts d_hits and the class planes
  // d_bits ([3][classes][Npad/32]: pass, E, A) are built on the device when dirty.  d_fipf: each fit class's filter
  // class, d_reasons the companion rows [P][3].  The placed side (bs_upload_pod_interpod_placed; dropped with the pod
  // table): each pod's placed class d_qclass [P] and the class table, what an assumed pod adds to presence in the walks;
  // placed_term_max is checked against node.terms when a walk starts.  walk_prepass: a walk ran the pre-pass, so the
  // next evaluation builds the class fit bits and gates again.
  struct {
    bool on = false, round = false;
    InterpodNodeSide node;
    DevBuf d_presence, d_hits, d_poff, d_pterm, d_prole, d_pself, d_bits, d_fipf, d_reasons;
    DevBuf d_qclass, d_qoff, d_qterm, d_qown, d_qmatch;
    bool have_node = false, have_pod = false, have_placed = false, dirty = true, walk_prepass = false;
    uint32_t pclasses = 0;
    int64_t term_max = -1, placed_term_max = -1;
    std::vector<uint32_t> h_class;
  } ipf;
  // PodFitsHostPorts filter (bs_set_host_port_filter; off by default): the node side (each entry's conflict mask
  // h_conflict, each node's used mask d_used [Npad]; dropped with the node table) and the pod side (each pod's want
  // mask h_want, want_all their OR; dropped with the pod table).  dirty: the used masks changed or the filter was
  // switched on, so the class fit bits are built again.  d_fconf: each fit class's conflict mask, d_bins the ports bin
  // of each fit class, d_reasons the companion rows [P].  The bound side (bs_upload_bound_host_ports; dropped with the
  // bound-pod table): each bound row's mask h_bports in table order, d_bports / d_bsuf the masks in CSR order and their
  // suffix OR; h_used keeps the node side's used masks for its checks.
  struct {
    bool on = false, round = false;
    DevBuf d_used, d_fconf, d_bins, d_reasons;
    bool have_node = false, have_pod = false, dirty = true, have_bound = false;
    uint32_t entries = 0;
    uint64_t want_all = 0;
    std::vector<uint64_t> h_conflict, h_want, h_used, h_bports;
    DevBuf d_bstage, d_bports, d_bsuf, d_pconf;   // d_pconf: bs_preempt's per-preemptor conflict masks
  } hp;
  // The filters' share of the fit classes.  assign_dirty: the pods' fit classes have to be assigned again (with their
  // filter class and conflict mask while a filter is on, else their base class h_pfc_base).  d_gate: the priority
  // lists' gate while a filter is on, the reason gate ANDed with the filters' pass bits.
  struct {
    bool assign_dirty = false;
    std::vector<uint32_t> h_pfc_base;   // the pods' fit classes without the filters
    bool pfc_base_valid = false;        // h_pfc_base holds the classes of the pod table of now
    DevBuf d_gate;
  } filt;
  // sort scratch: views into one arena
  View d_gk0, d_gk1, d_pk0, d_pk1, d_idx_a, d_idx_b, d_ghist, d_group_rank, d_tilecnt, d_sort_barrier;
  uint32_t sort_max_grid = 1;
  DevBuf d_sort_arena;
  // what the last round's sort launched (bs_sort_shape): kernel 0 none, 1 single-CTA, 2 persistent lean, 3 persistent wide
  struct SortShape { bool valid = false; uint32_t kernel = 0, grid = 0, group_passes = 0, pod_passes = 0; } sort_shape;
  // the regime of the last bs_replay / bs_replay_priority walk (bs_replay_shape)
  struct ReplayShape {
    bool valid = false;
    uint32_t cached = 0, fitmask = 0, n_rep = 0, n_blocks = 0, bucket_size = 0, n_buckets = 0, lo = 0, monotone = 0;
  } replay_shape;

  // host copies for the per-call mirrors and class building
  std::vector<int32_t> h_gid, h_prio;
  std::vector<uint8_t> h_pflags;
  std::vector<uint64_t> h_gsel, h_gtol;
  std::vector<uint8_t> h_nflags;
  // class indices (host packing): fit classes (sel, tol, nz) of the pods; representative classes
  // (sel, tol) of pods and carried-in group representatives
  ClassIndex fit_index, rep_index;
  PinVec<uint32_t> h_pfc, h_prc, h_grc;   // pinned: DMA'd whenever the classes change
  Event ev_classes;                       // the last class-table DMA out of them
  bool group_classes_dirty = true;   // every group's representative id has to be looked up again
  bool group_ids_dirty = false;      // some ids in h_grc changed in place (bs_update_groups): DMA them again
  std::vector<int64_t> h_wait_ns;
  int64_t default_wait_ns = 0;
  bool pod_classes_dirty = true;
  double last_classes_us = 0;
  // BS_HOST_PROFILE: host-side segment times (label, us) since the last bs_evaluate, printed there
  bool host_prof = false;
  std::vector<std::pair<const char*, double>> hp_log;
  std::chrono::steady_clock::time_point hp_t;
  // decision arena: every per-round decision vector lives in ONE device block and ONE pinned block with the
  // same layout (d_* views, and their h_* pinned mirrors), so bs_fetch is a single D2H copy
  View d_state, d_prefilter, d_feasible, d_best_node, d_best_score, d_admit, d_admit_bitmap, d_new_denied, d_order,
      d_rank, d_filter_code;
  View h_state, h_prefilter, h_feasible, h_best_node, h_best_score, h_admit, h_admit_bitmap, h_new_denied, h_order,
      h_rank, h_filter_code;
  DevBuf d_arena;
  PinBuf h_arena;
  size_t arena_bytes = 0;
  bool fetched = false;

  // bs_replay scratch (kept between calls: an allocation per call would dominate small queues)
  DevBuf d_replay;

  // bound-pod table (bs_upload_bound_pods): CSR by node in MoreImportantPod order, its suffix sums and counts, and
  // the residuals it is read against (node_left_kernel's full-width table, kept apart from the round's); dropped
  // with the node snapshot and with the group table
  bool have_bound = false;
  uint32_t V = 0;
  int32_t bound_max_gid = -1;
  std::vector<int32_t> h_bgid;        // by bound-table index: bs_remove_pod
  std::vector<uint32_t> h_bnode;      // by bound-table index: the bound host-port checks
  std::vector<uint8_t> h_bflags;
  std::vector<int32_t> h_npc;         // node pod_count and req_present as uploaded (bound-table validation)
  std::vector<uint32_t> h_nrpres;
  DevBuf d_brow, d_bprio, d_bstart, d_bgid, d_bflags, d_bidx, d_breq, d_bsuf, d_bsuf_online, d_bsuf_bad, d_bsuf_vio;
  DevBuf d_pl_left, d_pl_present;
  // bs_preempt scratch
  DevBuf d_pp, d_ptiles, d_pnode, d_pnv, d_pcand, d_poff, d_pvict;
  // bs_preempt_walk scratch: the live copies of the node and bound state, the outputs and the undo log
  DevBuf d_walk;

  // peer exchange (admit bitmap all-gather over NVLink peer memory)
  DevBuf d_gather, d_peer_err;
  uint32_t peer_rank = 0, peer_world = 0, peer_wpr = 0, peer_seq = 0;
  bool peer_attached = false;
  bool peer_broken = false;          // a wait timed out: every later round fails fast until detach + re-attach
  unsigned long long peer_timeout_ns = 2000000000ull;
  void* peer_ptr[PEER_MAX_WORLD] = {};

  // profiling
  bool profiling = false;
  Event ev_a[BS_K_COUNT], ev_b[BS_K_COUNT];
  uint32_t k_launches[BS_K_COUNT] = {};
  bool k_valid[BS_K_COUNT] = {};
};

namespace {

#define CK(call)                                                                     \
  do {                                                                               \
    cudaError_t _e = (call);                                                         \
    if (_e != cudaSuccess) {                                                         \
      e->err = std::string(#call) + ": " + cudaGetErrorString(_e);                   \
      cudaGetLastError();                                                            \
      return _e == cudaErrorMemoryAllocation ? BS_E_NOMEM : BS_E_CUDA;               \
    }                                                                                \
  } while (0)

int fail(bs_engine* e, int code, const char* msg) {
  e->err = msg;
  return code;
}

// Everything bs_upload_nodes / bs_update_nodes need from the N rows of host columns, in ONE chunked pass.
NodeStats node_host_pass(const bs_node_table* t, uint32_t L, uint32_t N) {
  return Chunks(N, 4096).reduce<NodeStats>([&](int, uint32_t a0, uint32_t a1, NodeStats& st) {
    for (uint32_t d = 0; d < L; ++d) {
      const int64_t* al = t->alloc + (size_t)d * N;
      const int64_t* rq = t->requested + (size_t)d * N;
      int64_t alo = 0, ahi = 0, rlo = 0, rhi = 0, mx = 0;
      uint64_t o = 0;
      for (uint32_t i = a0; i < a1; ++i) {
        alo = std::min(alo, al[i]); ahi = std::max(ahi, al[i]);
        rlo = std::min(rlo, rq[i]); rhi = std::max(rhi, rq[i]);
      }
      // (float)alloc is the RN convert, * 1.0f is exact, the cast back truncates: the device's scale_f32
      for (uint32_t i = a0; i < a1; ++i) {
        if (d >= 4 && !((t->alloc_present[i] & t->req_present[i]) >> d & 1u)) continue;   // key absent: sentinel
        int64_t used = rq[i];
        if (d == (uint32_t)LANE_PODS && used == 0) used = t->pod_count[i];
        const int64_t v = (int64_t)((float)al[i] * 1.0f) - used;
        o |= (uint64_t)v;
        mx = std::max(mx, v < 0 ? -v : v);
      }
      st.bad_range = st.bad_range || alo < -BS_VALUE_LIMIT || ahi > BS_VALUE_LIMIT || rlo < -BS_VALUE_LIMIT ||
                     rhi > BS_VALUE_LIMIT;
      st.max_alloc[d] = std::max(ahi, alo == INT64_MIN ? INT64_MAX : -alo);
      st.max_requested[d] = std::max(rhi, rlo == INT64_MIN ? INT64_MAX : -rlo);
      st.or_left[d] = o;
      st.max_left[d] = mx;
    }
    int64_t pc = 0;
    for (uint32_t i = a0; i < a1; ++i) pc = std::max<int64_t>(pc, std::abs((int64_t)t->pod_count[i]));
    st.max_pod_count = pc;
  });
}

// Everything bs_upload_groups / bs_update_groups need from the n rows of host columns, in ONE chunked pass: the
// |min_res| range, the creation sentinel, the OR / AND of the sort-key words and, with `reps` (an engine whose
// representative columns have n rows), whether the table's representative columns differ from that engine's.
GroupStats group_host_pass(const bs_group_table* t, uint32_t L, uint32_t n, const bs_engine* reps) {
  return Chunks(n, 8192).reduce<GroupStats>([&](int, uint32_t g0, uint32_t g1, GroupStats& st) {
    for (uint32_t d = 0; d < L; ++d) {
      const int64_t* row = t->min_res + (size_t)d * n;
      int64_t lo = 0, hi = 0;
      for (uint32_t g = g0; g < g1; ++g) { lo = std::min(lo, row[g]); hi = std::max(hi, row[g]); }
      st.bad_range = st.bad_range || lo < -BS_VALUE_LIMIT || hi > BS_VALUE_LIMIT;
    }
    uint64_t lo1 = 0, la1 = ~0ull, lo0 = 0, la0 = ~0ull;
    bool bc = false;
    for (uint32_t g = g0; g < g1; ++g) {
      const uint64_t c = (uint64_t)t->creation_ns[g], nm = (uint64_t)(~t->name_rank[g]);
      lo1 |= c; la1 &= c; lo0 |= nm; la0 &= nm;
      bc = bc || t->creation_ns[g] == INT64_MAX;
    }
    st.or_creation = lo1; st.and_creation = la1; st.or_name = lo0; st.and_name = la0; st.bad_creation = bc;
    if (reps && g1 > g0) {
      const size_t k = g1 - g0;
      bool df = memcmp(reps->h_gsel.data() + g0, t->rep_sel + g0, k * 8) != 0 ||
                memcmp(reps->h_gtol.data() + g0, t->rep_tol + g0, k * 8) != 0;
      const uint32_t* ha = reps->h_gaff.data();
      if (t->rep_aff_class) df = df || memcmp(ha + g0, t->rep_aff_class + g0, k * 4) != 0;
      else
        for (uint32_t g = g0; g < g1 && !df; ++g) df = ha[g] != BS_AFF_NONE;
      st.reps_differ = df;
    }
  });
}

// Lane classification for the fit kernel (kernels.cuh "Narrow lanes"): lane d is narrow when every
// residual |left[d]| and every request |req[d]| of the round is <= 2^27.  The narrow set must
// contain a fixed lane (always a real value) and the (LW, LN) pair must be one the dispatch
// table instantiates; otherwise every lane is wide.
LaneMap classify_lanes(const bs_engine* e);

inline uint32_t cdiv(uint32_t a, uint32_t b) { return (a + b - 1) / b; }

// A table column: the caller's host column ([lanes][rows]) and the resident device column ([lanes][padded rows]).
struct Col {
  const void* host;
  DevBuf* dev;
  uint32_t elem, lanes;   // element bytes, lanes
};
template <class T>
Col col(const T* host, DevBuf& dev, uint32_t lanes = 1) { return Col{host, &dev, (uint32_t)sizeof(T), lanes}; }

// the columns bs_upload_nodes / bs_update_nodes move to the device
std::array<Col, 8> node_cols(bs_engine* e, const bs_node_table* t) {
  return {col(t->alloc, e->d_alloc, e->L), col(t->requested, e->d_requested, e->L), col(t->pod_count, e->d_pod_count),
          col(t->alloc_present, e->d_apres), col(t->req_present, e->d_rpres), col(t->label_mask, e->d_label),
          col(t->taint_mask, e->d_taint), col(t->flags, e->d_nflags)};
}
// the columns bs_upload_groups / bs_update_groups move to the device (the representative columns stay on the host)
std::array<Col, 8> group_cols(bs_engine* e, const bs_group_table* t) {
  return {col(t->min_member, e->d_min_member), col(t->scheduled, e->d_scheduled), col(t->matched, e->d_matched),
          col(t->flags, e->d_gflags), col(t->min_res, e->d_min_res, e->L), col(t->min_res_present, e->d_mrpres),
          col(t->creation_ns, e->d_creation), col(t->name_rank, e->d_name_rank)};
}
template <size_t K>
bool null_column(const std::array<Col, K>& cols) {
  return std::any_of(cols.begin(), cols.end(), [](const Col& c) { return !c.host; });
}

// upload a host column of n rows into its device column padded to npad >= n rows (at least one allocated), the
// padding's bytes set to fill
int upload_col(bs_engine* e, const Col& c, uint64_t n, uint64_t npad, int fill = 0) {
  const size_t row = (size_t)c.elem * n, prow = (size_t)c.elem * npad;
  CK(c.dev->ensure((size_t)c.elem * std::max<uint64_t>(npad, 1) * c.lanes));
  if (npad > n) CK(cudaMemsetAsync(c.dev->p, fill, prow * c.lanes, e->s));
  if (n && c.lanes == 1) CK(cudaMemcpyAsync(c.dev->p, c.host, row, cudaMemcpyHostToDevice, e->s));
  else if (n) CK(cudaMemcpy2DAsync(c.dev->p, prow, c.host, row, row, c.lanes, cudaMemcpyHostToDevice, e->s));
  return BS_OK;
}
template <size_t K>
int upload_cols(bs_engine* e, const std::array<Col, K>& cols, uint32_t n, uint32_t npad) {
  int rc;
  for (const Col& c : cols)
    if ((rc = upload_col(e, c, n, npad))) return rc;
  return BS_OK;
}
template <class T>
int upload_vec(bs_engine* e, DevBuf& dst, const T* src, uint64_t n, uint64_t npad, int fill = 0) {
  return upload_col(e, col(src, dst), n, npad, fill);
}

// The largest class col[0, n) names, `none` aside (-1 when there is none).
int64_t max_class(const uint32_t* col, uint32_t n, uint32_t none) {
  int64_t mx = -1;
  for (uint32_t k = 0; k < n; ++k)
    if (col[k] != none) mx = std::max(mx, (int64_t)col[k]);
  return mx;
}

// A refusal of the call `who`: its code, with "who: why" as the engine's last error.
enum SideOf { NODE_SIDE, POD_SIDE };
struct Refuse {
  bs_engine* e;
  const char* who;
  int operator()(int rc, const char* why) const { return fail(e, rc, (std::string(who) + ": " + why).c_str()); }
  // a side table's shape: the table it belongs to is uploaded (BS_E_STATE) and has n rows (BS_E_INVAL)
  int shape(SideOf side, uint32_t n) const {
    if (side == NODE_SIDE && !e->have_nodes) return (*this)(BS_E_STATE, "upload nodes first");
    if (side == POD_SIDE && !e->have_pods) return (*this)(BS_E_STATE, "upload pods first");
    if (side == NODE_SIDE && n != e->N) return (*this)(BS_E_INVAL, "n_nodes differs from the node table's");
    if (side == POD_SIDE && n != e->P) return (*this)(BS_E_INVAL, "n_pods differs from the pod table's");
    return BS_OK;
  }
};

// Stages the n changed rows of every column, and idx, in d_stage, and scatters row k of each column to row
// idx[k] of its device column (pitch rows per lane).  The caller synchronises before its arrays are reused.
template <size_t K>
int scatter_rows(bs_engine* e, const std::array<Col, K>& cols, const uint32_t* idx, uint32_t n, uint32_t pitch) {
  static_assert(K <= SCATTER_MAX_COLS, "one ScatterCols slot per column");
  View stage[K + 1];
  Field fields[K + 1];
  for (size_t c = 0; c < K; ++c) fields[c] = Field{&stage[c], (size_t)cols[c].elem * cols[c].lanes * n};
  fields[K] = Field{&stage[K], (size_t)n * 4};
  CK(carve(e->d_stage, fields));
  ScatterCols sc{};
  sc.n_cols = K;
  for (size_t c = 0; c < K; ++c) {
    CK(cudaMemcpyAsync(stage[c].p, cols[c].host, stage[c].bytes, cudaMemcpyHostToDevice, e->s));
    sc.dst[c] = static_cast<uint8_t*>(cols[c].dev->p);
    sc.src[c] = static_cast<const uint8_t*>(stage[c].p);
    sc.elem[c] = cols[c].elem;
    sc.lanes[c] = cols[c].lanes;
  }
  CK(cudaMemcpyAsync(stage[K].p, idx, stage[K].bytes, cudaMemcpyHostToDevice, e->s));
  row_scatter_kernel<<<cdiv(n, 256), 256, 0, e->s>>>(sc, pitch, static_cast<const uint32_t*>(stage[K].p), n);
  e->launches++;
  return BS_OK;
}

NodeTab node_tab(const bs_engine* e) {
  NodeTab t;
  t.alloc = e->d_alloc.as<int64_t>();
  t.requested = e->d_requested.as<int64_t>();
  t.pod_count = e->d_pod_count.as<int32_t>();
  t.alloc_present = e->d_apres.as<uint32_t>();
  t.req_present = e->d_rpres.as<uint32_t>();
  t.label = e->d_label.as<uint64_t>();
  t.taint = e->d_taint.as<uint64_t>();
  t.flags = e->d_nflags.as<uint8_t>();
  t.aff_bits = e->d_aff_bits.as<uint32_t>();
  t.aff_W = e->W;
  t.N = e->N;
  t.Npad = e->Npad;
  t.L = e->L;
  return t;
}
PodTab pod_tab(const bs_engine* e) {
  PodTab p;
  p.req = e->d_req.as<int64_t>();
  p.req_present = e->d_ppres.as<uint32_t>();
  p.gid = e->d_gid.as<int32_t>();
  p.flags = e->d_pflags.as<uint8_t>();
  p.fit_class = e->d_pod_fit_class.as<uint32_t>();
  p.rep_class = e->d_pod_rep_class.as<uint32_t>();
  p.P = e->P;
  p.L = e->L;
  return p;
}
GroupTab group_tab(const bs_engine* e) {
  GroupTab g;
  g.min_member = e->d_min_member.as<uint32_t>();
  g.scheduled = e->d_scheduled.as<uint32_t>();
  g.matched = e->d_matched.as<uint32_t>();
  g.flags = e->d_gflags.as<uint8_t>();
  g.min_res = e->d_min_res.as<int64_t>();
  g.min_res_present = e->d_mrpres.as<uint32_t>();
  g.rep_class = e->d_group_rep_class.as<uint32_t>();
  g.G = e->G;
  g.L = e->L;
  return g;
}
GroupEff group_eff(const bs_engine* e) {
  GroupEff x;
  x.flags = e->d_eflags.as<uint8_t>();
  x.min_res = e->d_emin_res.as<int64_t>();
  x.min_res_present = e->d_emrpres.as<uint32_t>();
  x.rep_class = e->d_erep_class.as<uint32_t>();
  x.first_pod = e->d_first_pod.as<uint32_t>();
  x.in_round = e->d_in_round.as<uint32_t>();
  x.contrib = e->d_contrib.as<uint32_t>();
  x.done = e->d_done.as<uint32_t>();
  return x;
}
PrefixOut prefix_out(const bs_engine* e) {
  PrefixOut o;
  o.pre = e->d_pre.as<int64_t>();
  o.present = e->d_pre_present.as<uint32_t>();
  o.stats = e->d_pre_stats.as<ClassStats>();
  return o;
}

PrefixScratch prefix_scratch(const bs_engine* e) {
  PrefixScratch sc;
  sc.part = e->d_pre_part.as<int64_t>();
  sc.part_pres = e->d_pre_part_pres.as<uint32_t>();
  sc.cstats = e->d_pre_cstats.as<ClassStats>();
  sc.done = e->d_pre_done.as<uint32_t>();
  return sc;
}

// Makes the engine's device current for the scope and restores the caller's device afterwards
// (the library must not leave the calling thread on a different device).
struct DeviceGuard {
  int prev = -1;
  cudaError_t err = cudaSuccess;
  explicit DeviceGuard(int dev) {
    if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
    if (prev != dev) err = cudaSetDevice(dev);
  }
  ~DeviceGuard() {
    int cur = -1;
    if (prev >= 0 && cudaGetDevice(&cur) == cudaSuccess && cur != prev) cudaSetDevice(prev);
  }
};
#define BS_DEVICE_GUARD(e)        \
  DeviceGuard _guard((e)->device); \
  CK(_guard.err)

// host-side segment timer (BS_HOST_PROFILE): HP_BEGIN at the top of an entry point, HP("what") after a segment
#define HP_BEGIN(e) do { if ((e)->host_prof) (e)->hp_t = std::chrono::steady_clock::now(); } while (0)
#define HP(e, label) do { if ((e)->host_prof) { const auto _n = std::chrono::steady_clock::now(); \
    if ((e)->hp_log.size() > 4096) (e)->hp_log.clear(); (e)->hp_log.emplace_back(label, std::chrono::duration<double, std::micro>(_n - (e)->hp_t).count()); (e)->hp_t = _n; } } while (0)

struct StageTimer {
  bs_engine* e;
  int k;
  cudaStream_t st;
  bool manual;   // the launcher records the two events itself (gang_fit: around the one kernel)
  StageTimer(bs_engine* e_, int k_, cudaStream_t st_, bool manual_ = false) : e(e_), k(k_), st(st_), manual(manual_) {
    e->k_launches[k] = 0;
    if (e->profiling && !manual) cudaEventRecord(e->ev_a[k], st);
  }
  ~StageTimer() {
    if (e->profiling && !manual) {
      cudaEventRecord(e->ev_b[k], st);
      e->k_valid[k] = true;
    }
  }
  void launched(uint32_t n = 1) {
    e->k_launches[k] += n;
    e->launches += n;
  }
};

// two launches: chunk totals, then offsets + in-chunk scan + statistics
void launch_prefix(uint32_t L, NodeTab t, PrefixSel ps, PrefixScratch sc, PrefixOut po, uint32_t n_classes,
                   cudaStream_t s) {
  const uint32_t n_chunks = cdiv(t.N, PREFIX_CHUNK);
  dim3 grid(n_chunks, n_classes);
  with_maxl<4, 5, 6, 8, 9, 12, 16>(L, [&](auto M) {
    prefix_partial_kernel<M><<<grid, PREFIX_CHUNK, 0, s>>>(t, ps, sc, n_chunks);
    prefix_scan_kernel<M><<<grid, PREFIX_CHUNK, 0, s>>>(t, ps, sc, n_chunks, po);
  });
}

// priority.cuh: the build of priority_pod_kernel for L lanes and `terms` (PRIO_*)
cudaError_t launch_priority(uint32_t L, uint32_t grid, uint32_t terms, const PriorityIpaArgs& a, cudaStream_t s) {
  with_maxl<5, 9, 16>(L, [&](auto M) {
    (terms & PRIO_IPA ? launch_priority_slice<M, PRIO_IPA> : launch_priority_slice<M, 0>)(terms, grid, a, s);
  });
  return cudaGetLastError();
}

// replay.cuh: the build of replay_kernel for L lanes and `build` (REPLAY_*)
void launch_replay(uint32_t L, uint32_t build, const ReplayIpfArgs& a, cudaStream_t s) {
  with_maxl<5, 9, 16>(L, [&](auto M) {
    (build & REPLAY_IPF ? launch_replay_slice<M, REPLAY_IPF> : launch_replay_slice<M, 0>)(build, a, s);
  });
}

cudaError_t launch_fit(const FitArgs& a, uint32_t units, cudaStream_t s, uint32_t* launches, cudaEvent_t ev_a, cudaEvent_t ev_b) {
  const int out = a.score ? FIT_OUT_SCORE : a.topk_node ? FIT_OUT_TOPK : a.fit_bitmap ? FIT_OUT_BITMAP : FIT_OUT_NONE;
  FitFn fn = fit_lookup(a.lm.LW, a.lm.LN, a.lm.LS, out);
  return fn ? fn(a, units, s, launches, ev_a, ev_b) : cudaErrorInvalidValue;
}

inline uint32_t ctz64(uint64_t v) { return v ? (uint32_t)__builtin_ctzll(v) : 63u; }

LaneMap classify_lanes(const bs_engine* e) {
  LaneMap lm{};
  const uint32_t L = e->L;
  enum { WIDE = 0, NARROW = 1, SCALED = 2 };
  int kind[BS_MAX_LANES];
  uint32_t unit[BS_MAX_LANES] = {};
  bool fixed_narrow = false;
  uint32_t ln = 0, ls = 0;
  const NodeStats& ns = e->node_stats;
  const PodStats& ps = e->pod_stats;
  for (uint32_t d = 0; d < L; ++d) {
    // |left| <= |scale(alloc)| + |requested| (pods lane: + len(Pods())); float32 rounding of a
    // value <= 2^26 is exact, so the bound 2^26 + 2^26 = 2^27 holds.
    int64_t used = ns.max_requested[d];
    if (d == LANE_PODS) used = std::max(used, ns.max_pod_count);
    const bool narrow = ns.max_alloc[d] <= (NARROW_LIMIT >> 1) && used <= (NARROW_LIMIT >> 1) && ps.max_req[d] <= NARROW_LIMIT;
    kind[d] = narrow ? NARROW : WIDE;
    if (narrow) {
      ++ln;
      if (d < 4) fixed_narrow = true;
      continue;
    }
    // scaled: every residual and every request of the lane is a multiple of 2^k (k from the OR of all
    // values seen at upload) and fits 2^29 in those units; the smallest such k is taken
    const uint32_t k_avail = std::min(ctz64(ns.or_left[d]), ctz64(ps.or_req[d]));
    const int64_t mx = std::max(ns.max_left[d], ps.max_req[d]);
    uint32_t k_need = 0;
    while (k_need < 63 && (mx >> k_need) > SCALED_LIMIT) ++k_need;
    if (k_need <= k_avail) {
      kind[d] = SCALED;
      unit[d] = k_need;
      ++ls;
    }
  }
  // keep at most FIT_MAX_LN narrow lanes (prefer the fixed ones)
  if (fixed_narrow && ln > (uint32_t)FIT_MAX_LN)
    for (int d = (int)L - 1; d >= 4 && ln > (uint32_t)FIT_MAX_LN; --d)
      if (kind[d] == NARROW) { kind[d] = WIDE; --ln; }
  // scaled lanes back to wide (last first) until the shape is one the variant table holds
  if (fixed_narrow) {
    for (int d = (int)L - 1; d >= 0 && !fit_variant_exists(L - ln - ls, ln, ls) && ls > 0; --d)
      if (kind[d] == SCALED) { kind[d] = WIDE; --ls; }
  }
  if (!fixed_narrow || !fit_variant_exists(L - ln - ls, ln, ls)) {
    for (uint32_t d = 0; d < L; ++d) kind[d] = WIDE;
    ln = ls = 0;
  }
  for (uint32_t d = 0; d < L; ++d) {
    if (kind[d] == NARROW) lm.narrow[lm.LN++] = (uint8_t)d;
    else if (kind[d] == SCALED) {
      const uint32_t k = unit[d];
      lm.scaled[lm.LS] = (uint8_t)d;
      lm.sunit[lm.LS] = (uint8_t)k;
      lm.sshift[lm.LS] = (uint8_t)std::min(k, (uint32_t)FIT_CAP_LOG2);
      lm.sclamp[lm.LS] = k <= (uint32_t)FIT_CAP_LOG2 ? (1u << (FIT_CAP_LOG2 - k)) : 1u;
      ++lm.LS;
    } else lm.wide[lm.LW++] = (uint8_t)d;
  }
  return lm;
}

// radix passes for the byte digits of (k0, k1) that actually vary (LSD order: k0 low..high, k1 low..high)
uint32_t build_passes(uint64_t vary0, uint64_t vary1, SortPass* out) {
  uint32_t n = 0;
  for (int sh = 0; sh < 64; sh += 8)
    if ((vary0 >> sh) & 0xffull) out[n++] = SortPass{0, (uint8_t)sh};
  for (int sh = 0; sh < 64; sh += 8)
    if ((vary1 >> sh) & 0xffull) out[n++] = SortPass{1, (uint8_t)sh};
  return n;
}

inline uint64_t low_bits_mask(uint32_t n) {  // mask covering every value in [0, n]
  uint64_t m = 0;
  while (m < n) m = (m << 1) | 1ull;
  return m;
}

// The fit index only grows.  While a filter is on, every side upload and every switch adds (class, filter class,
// conflict mask) keys, so after each re-assignment the index is rebuilt from the classes the pods use when those are a
// small share of it (the bound bs_upload_pods applies to stale classes); the base ids of h_pfc_base follow.
void compact_fit_index(bs_engine* e) {
  ClassIndex& fi = e->fit_index;
  const uint32_t P = e->P;
  uint32_t* pfc = e->h_pfc.data();
  uint32_t* base = e->filt.pfc_base_valid ? e->filt.h_pfc_base.data() : nullptr;
  std::vector<uint8_t> used(fi.size(), 0);
  size_t n_used = 0;
  auto mark = [&](uint32_t id) { n_used += used[id] ? 0 : 1; used[id] = 1; };
  for (uint32_t p = 0; p < P; ++p) {
    mark(pfc[p]);
    if (base) mark(base[p]);
  }
  if (fi.size() <= std::max<size_t>(4096, 4 * n_used)) return;
  ClassIndex ni;
  ni.clear();
  for (uint32_t p = 0; p < P; ++p) {
    if (base) base[p] = ni.get_or_add(fi.keys[base[p]]);
    pfc[p] = ni.get_or_add(fi.keys[pfc[p]]);
  }
  fi = std::move(ni);
}

// A PodFitsHostPorts want mask's conflict mask: the OR of the node side's conflict masks of the entries it wants.
uint64_t hp_conflict_of(const bs_engine* e, uint64_t want) {
  uint64_t conf = 0;
  for (; want; want &= want - 1) conf |= e->hp.h_conflict[__builtin_ctzll(want)];
  return conf;
}

int rebuild_classes(bs_engine* e) {
  // Pod classes were indexed while the pod table was uploaded; group representative classes are
  // looked up here (the representative index must already hold the pods' (sel, tol) pairs so that
  // the ids agree).  Then the class tables go to the device.
  const uint32_t P = e->P, G = e->G;
  HP_BEGIN(e);
  CK(cudaEventSynchronize(e->ev_classes));   // a previous DMA out of h_grc has finished
  HP(e, "classes:event-wait");
  const bool groups_assigned = e->group_classes_dirty;
  if (e->group_classes_dirty) {
    if (!e->h_grc.resize(G)) return fail(e, BS_E_NOMEM, "pinned host memory");
    const uint64_t* gs = e->h_gsel.data();
    const uint64_t* gt = e->h_gtol.data();
    const uint32_t* ga = e->h_gaff.data();
    assign_classes(e->rep_index, G, [=](uint32_t g) { return ClassKey{gs[g], gt[g], 0u, ga[g]}; }, e->h_grc.data());
    e->group_classes_dirty = false;
  }
  HP(e, "classes:assign-groups");
  if (e->filt.assign_dirty) {
    // the pods' fit classes with their filter class and conflict mask while a filter is on, else the classes of the
    // upload (the evaluation's checks have passed: both sides of each filter that is on are here and agree)
    uint32_t* pfc = e->h_pfc.data();
    if (e->ipf.on || e->hp.on) {
      if (!e->filt.pfc_base_valid) e->filt.h_pfc_base.assign(pfc, pfc + P);
      e->filt.pfc_base_valid = true;
      const uint32_t* base = e->filt.h_pfc_base.data();
      const uint32_t* ipf = e->ipf.on ? e->ipf.h_class.data() : nullptr;
      const uint64_t* want = e->hp.on ? e->hp.h_want.data() : nullptr;
      ClassIndex& fi = e->fit_index;
      assign_classes(fi, P, [e, &fi, base, ipf, want](uint32_t p) {
        ClassKey k = fi.keys[base[p]];
        if (ipf) k.ipf = ipf[p];
        if (want) k.hp |= hp_conflict_of(e, want[p]);
        return k;
      }, pfc);
    } else if (e->filt.pfc_base_valid) {
      memcpy(pfc, e->filt.h_pfc_base.data(), (size_t)P * 4);
    }
    compact_fit_index(e);
    e->filt.assign_dirty = false;
  }
  if (e->fit_index.size() == 0) e->fit_index.get_or_add(ClassKey{0, 0, 0, BS_AFF_NONE});
  if (e->rep_index.size() == 0) e->rep_index.get_or_add(ClassKey{0, 0, 0, BS_AFF_NONE});
  e->n_fit_classes = (uint32_t)e->fit_index.size();
  e->n_rep_classes = (uint32_t)e->rep_index.size();
  std::vector<uint64_t> fsel(e->n_fit_classes), ftol(e->n_fit_classes), rsel(e->n_rep_classes), rtol(e->n_rep_classes);
  std::vector<uint32_t> fnz(e->n_fit_classes), faff(e->n_fit_classes), raff(e->n_rep_classes);
  bool aff_bad = false, any_aff = false;
  // Stale classes of earlier tables linger in both persistent indices and may name an affinity row the table of now
  // does not have.  Only the classes in use are checked: a pod's fit and representative class carry its own affinity
  // id and a group's representative class the group's, so the pods and groups below are checked, not the indices.  A
  // stale class's bits are never read, so its out-of-range id goes to the device as no constraint: no kernel ever
  // indexes the table with it (the walk's fit mask covers every representative class).
  auto aff_row = [e](uint32_t a) { return a != BS_AFF_NONE && a >= e->n_aff ? BS_AFF_NONE : a; };
  for (uint32_t c = 0; c < e->n_fit_classes; ++c) {
    fsel[c] = e->fit_index.keys[c].sel; ftol[c] = e->fit_index.keys[c].tol; fnz[c] = e->fit_index.keys[c].nz;
    faff[c] = aff_row(e->fit_index.keys[c].aff);
  }
  for (uint32_t c = 0; c < e->n_rep_classes; ++c) {
    rsel[c] = e->rep_index.keys[c].sel; rtol[c] = e->rep_index.keys[c].tol; raff[c] = aff_row(e->rep_index.keys[c].aff);
    any_aff = any_aff || e->rep_index.keys[c].aff != BS_AFF_NONE;
  }
  if (any_aff) {   // else no pod or group names an affinity class: nothing to check
    for (uint32_t p = 0; p < P && !aff_bad; ++p) {
      const uint32_t a = e->rep_index.keys[e->h_prc[p]].aff;
      aff_bad = a != BS_AFF_NONE && a >= e->n_aff;
    }
    for (uint32_t g = 0; g < G && !aff_bad; ++g) aff_bad = e->h_gaff[g] != BS_AFF_NONE && e->h_gaff[g] >= e->n_aff;
  }
  if (aff_bad) {
    if (groups_assigned) e->group_classes_dirty = true;   // their ids were not uploaded: assign again next time
    // (group_ids_dirty stays set: an in-place change is uploaded by the next successful rebuild)
    return fail(e, BS_E_INDEX, "affinity class outside the uploaded table (bs_upload_affinity after bs_upload_nodes)");
  }
  HP(e, "classes:tables+checks");
  int rc;
  // cudaMemcpyAsync from pageable memory returns once the data is staged, so the vectors may die.
  if ((rc = upload_vec(e, e->d_fsel, fsel.data(), e->n_fit_classes, e->n_fit_classes))) return rc;
  if ((rc = upload_vec(e, e->d_ftol, ftol.data(), e->n_fit_classes, e->n_fit_classes))) return rc;
  if ((rc = upload_vec(e, e->d_fnz, fnz.data(), e->n_fit_classes, e->n_fit_classes))) return rc;
  if ((rc = upload_vec(e, e->d_faff, faff.data(), e->n_fit_classes, e->n_fit_classes))) return rc;
  if ((rc = upload_vec(e, e->d_raff, raff.data(), e->n_rep_classes, e->n_rep_classes))) return rc;
  if ((rc = upload_vec(e, e->d_rsel, rsel.data(), e->n_rep_classes, e->n_rep_classes))) return rc;
  if ((rc = upload_vec(e, e->d_rtol, rtol.data(), e->n_rep_classes, e->n_rep_classes))) return rc;
  if (e->ipf.on) {
    // a stale class may name a filter class the pod side of now does not have: no pod uses it, so it passes
    std::vector<uint32_t> fipf(e->n_fit_classes);
    for (uint32_t c = 0; c < e->n_fit_classes; ++c) {
      const uint32_t f = e->fit_index.keys[c].ipf;
      fipf[c] = f < e->ipf.pclasses ? f : BS_IPF_NONE;
    }
    if ((rc = upload_vec(e, e->ipf.d_fipf, fipf.data(), e->n_fit_classes, e->n_fit_classes))) return rc;
  }
  if (e->hp.on) {
    std::vector<uint64_t> fconf(e->n_fit_classes);
    for (uint32_t c = 0; c < e->n_fit_classes; ++c) fconf[c] = e->fit_index.keys[c].hp;
    if ((rc = upload_vec(e, e->hp.d_fconf, fconf.data(), e->n_fit_classes, e->n_fit_classes))) return rc;
  }
  if (e->pod_classes_dirty) {   // a group-only change (bs_update_groups) leaves the pods' ids alone
    if ((rc = upload_vec(e, e->d_pod_fit_class, e->h_pfc.data(), P, std::max(P, 1u)))) return rc;
    if ((rc = upload_vec(e, e->d_pod_rep_class, e->h_prc.data(), P, std::max(P, 1u)))) return rc;
  }
  if ((groups_assigned || e->group_ids_dirty) &&
      (rc = upload_vec(e, e->d_group_rep_class, e->h_grc.data(), G, std::max(G, 1u)))) return rc;
  e->group_ids_dirty = false;
  CK(cudaEventRecord(e->ev_classes, e->s));   // the pinned id arrays are read asynchronously from here on
  HP(e, "classes:uploads");
  e->classes_dirty = false;
  e->pod_classes_dirty = false;
  return BS_OK;
}

int ensure_round_buffers(bs_engine* e) {
  const uint32_t P = std::max(e->P, 1u), G = std::max(e->G, 1u), L = e->L, N = std::max(e->N, 1u);
  CK(e->d_eflags.ensure(G));
  CK(e->d_emin_res.ensure((size_t)L * G * 8));
  CK(e->d_emrpres.ensure((size_t)G * 4));
  CK(e->d_erep_class.ensure((size_t)G * 4));
  CK(e->d_first_pod.ensure((size_t)G * 4));
  CK(e->d_in_round.ensure((size_t)G * 4));
  CK(e->d_contrib.ensure((size_t)G * 4));
  CK(e->d_done.ensure((size_t)G * 4));
  CK(e->d_okA.ensure(G));
  CK(carve(e->d_arena,
           {{&e->d_state, sizeof(RoundState), &e->h_state},
            {&e->d_prefilter, P, &e->h_prefilter},
            {&e->d_feasible, (size_t)P * 4, &e->h_feasible},
            {&e->d_best_node, (size_t)P * 4, &e->h_best_node},
            {&e->d_best_score, (size_t)P * 8, &e->h_best_score},
            {&e->d_admit, G, &e->h_admit},
            {&e->d_admit_bitmap, (size_t)cdiv(G, 32) * 4, &e->h_admit_bitmap},
            {&e->d_new_denied, G, &e->h_new_denied},
            {&e->d_order, (size_t)P * 4, &e->h_order},
            {&e->d_rank, (size_t)P * 4, &e->h_rank},
            {&e->d_filter_code, (e->out_flags & BS_OUT_FILTER) ? (size_t)P : 0, &e->h_filter_code}},
           &e->h_arena, &e->arena_bytes));
  CK(e->d_best_packed.ensure((size_t)P * 8));
  // rows padded to a whole CTA of pods: the fit kernel writes pods >= P without a guard
  const size_t Prows = (size_t)cdiv(std::max(e->P, 1u), PODS_PER_CTA) * PODS_PER_CTA;
  if (e->out_flags & BS_OUT_FIT_BITMAP) CK(e->d_fit_bitmap.ensure(Prows * std::max(e->bitmap_pitch, 32u) * 4));
  if (e->out_flags & BS_OUT_SCORE) CK(e->d_score.ensure(Prows * std::max(e->score_pitch, 2u) * 8));
  if (e->out_flags & BS_OUT_TOPK) {
    CK(e->d_topk_node.ensure(Prows * e->topk * 4));
    CK(e->d_topk_score.ensure(Prows * e->topk * 8));
  }
  if (e->out_flags & BS_OUT_FILTER) {
    CK(e->d_filter_bitmap.ensure(Prows * std::max(e->W, 1u) * 4));
  }
  if (e->out_flags & BS_OUT_REASONS) CK(e->d_reasons.ensure((size_t)P * (4 + L) * 4));
  if ((e->out_flags & BS_OUT_REASONS) && e->ipf.on) CK(e->ipf.d_reasons.ensure((size_t)P * 3 * 4));
  if ((e->out_flags & BS_OUT_REASONS) && e->hp.on) CK(e->hp.d_reasons.ensure((size_t)P * 4));
  if (e->out_flags & BS_OUT_PRIORITY) {
    CK(e->d_prio_node.ensure((size_t)P * e->topk * 4));
    CK(e->d_prio_score.ensure((size_t)P * e->topk * 8));
  }
  // prefix scratch: as many rep-class slots as fit a 1 GiB budget
  const size_t per_class = (size_t)N * (8 * L + 4);
  // BS_PREFIX_BUDGET_BYTES (default 1 GiB) bounds the scratch; classes beyond it are processed in chunks
  size_t budget = (size_t)1 << 30;
  if (const char* bs = getenv("BS_PREFIX_BUDGET_BYTES")) budget = std::max<size_t>(1, strtoull(bs, nullptr, 10));
  uint32_t slots = (uint32_t)std::max<size_t>(1, std::min<size_t>(e->n_rep_classes, budget / per_class));
  slots = std::min(slots, 32768u);   // one grid row (gridDim.y <= 65535) per resident class
  e->prefix_slots = slots;
  CK(e->d_pre.ensure((size_t)slots * L * N * 8));
  CK(e->d_pre_present.ensure((size_t)slots * N * 4));
  CK(e->d_pre_stats.ensure((size_t)slots * sizeof(ClassStats)));
  {
    const size_t n_chunks = cdiv(N, PREFIX_CHUNK);
    const bool fresh = e->d_pre_done.cap < (size_t)slots * 4;
    CK(e->d_pre_part.ensure((size_t)slots * n_chunks * BS_MAX_LANES * 8));
    CK(e->d_pre_part_pres.ensure((size_t)slots * n_chunks * 4));
    CK(e->d_pre_cstats.ensure((size_t)slots * n_chunks * sizeof(ClassStats)));
    CK(e->d_pre_done.ensure((size_t)slots * 4));
    if (fresh) CK(cudaMemsetAsync(e->d_pre_done.p, 0, e->d_pre_done.cap, e->s));
    CK(e->d_max_partial.ensure((size_t)cdiv(G, FINDMAX_THREADS * FINDMAX_PER_THREAD) * sizeof(MaxState)));
  }
  // sort scratch: one arena.  No persisting-L2 window over it: the set-aside such a window needs cost the score-mode
  // gang_fit kernel 0.9 ms of 3.85 on an H100 (its 8 GB score stream through a smaller L2), and the sort was no
  // faster with it.
  const uint32_t M = std::max(P, G);
  CK(carve(e->d_sort_arena,
           {{&e->d_gk0, (size_t)G * 8}, {&e->d_gk1, (size_t)G * 8}, {&e->d_pk0, (size_t)P * 8}, {&e->d_pk1, (size_t)P * 8},
            {&e->d_idx_a, (size_t)M * 4}, {&e->d_idx_b, (size_t)M * 4},
            {&e->d_ghist, (size_t)3 * 256 * cdiv(M, SORT_TILE) * 4}, {&e->d_tilecnt, (size_t)cdiv(M, SORT_TILE) * 4},
            {&e->d_sort_barrier, sizeof(unsigned int)}, {&e->d_group_rank, (size_t)G * 4}}));
  return BS_OK;
}

int prepare_nodes(bs_engine* e) {
  // node_left + class fit bitmap (only when nodes or classes changed)
  NodeTab t = node_tab(e);
  StageTimer tm(e, BS_K_NODE_LEFT, e->s);
  CK(e->d_left_w.ensure((size_t)std::max(e->lane_map.LW, 1u) * e->Npad * 8));
  CK(e->d_left_n.ensure((size_t)std::max(e->lane_map.LN + e->lane_map.LS, 1u) * e->Npad * 4));
  CK(e->d_left_present.ensure((size_t)e->Npad * 4));
  if (e->out_flags & BS_OUT_FILTER) CK(e->d_left_plain.ensure((size_t)4 * e->Npad * 8));
  // the reason rows' residuals and gate bitmap: also the fit set of the priority lists
  const bool reasons = (e->out_flags & (BS_OUT_REASONS | BS_OUT_PRIORITY)) != 0;
  if (reasons) CK(e->d_left_full.ensure((size_t)e->L * e->Npad * 8));
  const uint32_t n_tiles = e->Npad / NODE_TILE;
  CK(e->d_classfit.ensure((size_t)e->n_fit_classes * n_tiles * 32 * sizeof(ColBits)));
  node_left_kernel<<<cdiv(e->Npad, 256), 256, 0, e->s>>>(t, e->lane_map, e->d_left_w.as<int64_t>(),
                                                         e->d_left_n.as<int32_t>(),
                                                         e->d_left_present.as<uint32_t>(),
                                                         (e->out_flags & BS_OUT_FILTER) ? e->d_left_plain.as<int64_t>() : nullptr,
                                                         reasons ? e->d_left_full.as<int64_t>() : nullptr);
  tm.launched();
  {
    for (uint32_t c0 = 0; c0 < e->n_fit_classes; c0 += 32768) {
      dim3 grid(cdiv(n_tiles * 32, 256), std::min(32768u, e->n_fit_classes - c0));
      auto fn = e->ipf.on ? (e->hp.on ? class_fit_kernel<true, true> : class_fit_kernel<true, false>)
                          : (e->hp.on ? class_fit_kernel<false, true> : class_fit_kernel<false, false>);
      fn<<<grid, 256, 0, e->s>>>(t, e->d_left_present.as<uint32_t>(), e->d_fsel.as<uint64_t>(), e->d_ftol.as<uint64_t>(),
                                 e->d_fnz.as<uint32_t>(), e->d_faff.as<uint32_t>(), e->n_fit_classes, n_tiles,
                                 e->d_classfit.as<ColBits>(), c0, e->ipf.d_fipf.as<uint32_t>(),
                                 e->ipf.d_bits.as<uint32_t>(), e->Npad / 32, e->hp.d_fconf.as<uint64_t>(),
                                 e->hp.d_used.as<uint64_t>());
      tm.launched();
    }
  }
  if (reasons) {
    // the class half of the reason rows follows the same inputs as the class fit bits
    const uint32_t Wg = e->Npad / 32;
    CK(e->d_reason_gate.ensure((size_t)e->n_fit_classes * Wg * 4));
    CK(e->d_reason_class.ensure((size_t)e->n_fit_classes * 4 * 4));
    CK(cudaMemsetAsync(e->d_reason_class.p, 0, (size_t)e->n_fit_classes * 4 * 4, e->s));
    if (e->ipf.on || e->hp.on) CK(e->filt.d_gate.ensure((size_t)e->n_fit_classes * Wg * 4));
    if (e->hp.on) {
      CK(e->hp.d_bins.ensure((size_t)e->n_fit_classes * 4));
      CK(cudaMemsetAsync(e->hp.d_bins.p, 0, (size_t)e->n_fit_classes * 4, e->s));
    }
    const HostPortClassArgs hpa{e->hp.d_fconf.as<uint64_t>(), e->hp.d_used.as<uint64_t>(), e->hp.d_bins.as<uint32_t>()};
    for (uint32_t c0 = 0; c0 < e->n_fit_classes; c0 += 32768) {
      dim3 grid(cdiv(Wg * 32, REASON_CLASS_THREADS), std::min(32768u, e->n_fit_classes - c0));
      auto fn = e->ipf.on ? (e->hp.on ? reason_class_kernel<true, true> : reason_class_kernel<true, false>)
                          : (e->hp.on ? reason_class_kernel<false, true> : reason_class_kernel<false, false>);
      fn<<<grid, REASON_CLASS_THREADS, 0, e->s>>>(t, e->d_fsel.as<uint64_t>(), e->d_ftol.as<uint64_t>(),
                                                  e->d_faff.as<uint32_t>(), e->n_fit_classes, Wg,
                                                  e->d_reason_gate.as<uint32_t>(), e->d_reason_class.as<uint32_t>(), c0,
                                                  e->ipf.d_fipf.as<uint32_t>(), e->ipf.d_bits.as<uint32_t>(),
                                                  e->filt.d_gate.as<uint32_t>(), hpa);
      tm.launched();
    }
  }
  CK(cudaGetLastError());
  e->nodes_dirty = false;
  return BS_OK;
}

// The side tables' checks before anything is launched: the columns a non-zero weight (or the filter switch) reads,
// BS_E_STATE when a side is missing, the ids they hold (BS_E_INDEX) and the tables they size (BS_E_INVAL).  The pod
// sides outlive node uploads: their class x node tables are checked against the node table of now.
int nonzero_check(bs_engine* e, const char* who) {
  if (!(e->nz.have_node && e->nz.have_pod))
    return Refuse{e, who}(BS_E_STATE, "BS_OUT_PRIORITY needs the node and pod non-zero columns");
  return BS_OK;
}

int preference_check(bs_engine* e, const char* who) {
  const Refuse bad{e, who};
  if (!(e->w_taint || e->w_naff)) return BS_OK;
  if (!(e->pref.have_node && e->pref.have_pod))
    return bad(BS_E_STATE, "a non-zero node priority weight needs the node and pod preference columns");
  if (e->w_naff && e->pref.class_max >= (int64_t)e->pref.classes)
    return bad(BS_E_INDEX, "a pod's preference class is outside the uploaded weight table");
  return BS_OK;
}

int locality_check(bs_engine* e, const char* who) {
  const Refuse bad{e, who};
  if (e->w_img) {
    if (!(e->loc.have_img_node && e->loc.have_img_pod))
      return bad(BS_E_STATE, "a non-zero ImageLocality weight needs the node and pod image columns");
    if (e->loc.class_max >= (int64_t)e->loc.classes)
      return bad(BS_E_INDEX, "a pod's image class is outside the uploaded classes");
    if (e->loc.image_max >= (int64_t)e->loc.images)
      return bad(BS_E_INDEX, "an image class lists an id outside the node side's image dictionary");
    if ((uint64_t)e->loc.classes * e->Npad > BS_LOC_TABLE_MAX_BYTES)
      return bad(BS_E_INVAL, "n_classes x padded nodes bytes exceeds BS_LOC_TABLE_MAX_BYTES");
  }
  if (e->w_avoid && !(e->loc.have_avoid_node && e->loc.have_avoid_pod))
    return bad(BS_E_STATE, "a non-zero NodePreferAvoidPods weight needs the node and pod avoid columns");
  return BS_OK;
}

int spread_check(bs_engine* e, const char* who) {
  const Refuse bad{e, who};
  if (!e->w_spread) return BS_OK;
  if (!(e->spread.have_node && e->spread.have_pod))
    return bad(BS_E_STATE, "a non-zero SelectorSpread weight needs the node and pod spread columns");
  if (e->spread.class_max >= (int64_t)e->spread.classes)
    return bad(BS_E_INDEX, "a pod's spread class is outside the uploaded count table");
  return BS_OK;
}

int interpod_check(bs_engine* e, const char* who) {
  const Refuse bad{e, who};
  if (!e->w_ipa) return BS_OK;
  if (!(e->ipa.have_node && e->ipa.have_pod))
    return bad(BS_E_STATE, "a non-zero InterPodAffinity weight needs the node and pod inter-pod sides");
  if (e->ipa.term_max >= (int64_t)e->ipa.node.terms)
    return bad(BS_E_INDEX, "a pod class's term is outside the node side's term dictionary");
  if ((uint64_t)e->ipa.pclasses * e->Npad * 8 > BS_IPA_TABLE_MAX_BYTES)
    return bad(BS_E_INVAL, "pod n_classes x padded nodes x 8 bytes exceeds BS_IPA_TABLE_MAX_BYTES");
  return BS_OK;
}

int interpod_filter_check(bs_engine* e, const char* who) {
  const Refuse bad{e, who};
  if (!(e->ipf.have_node && e->ipf.have_pod))
    return bad(BS_E_STATE, "the MatchInterPodAffinity filter needs its node and pod sides");
  if (e->ipf.term_max >= (int64_t)e->ipf.node.terms)
    return bad(BS_E_INDEX, "a filter class's term is outside the node side's term dictionary");
  if (3ull * e->ipf.pclasses * (e->Npad / 8) > BS_IPF_TABLE_MAX_BYTES)
    return bad(BS_E_INVAL, "3 x filter n_classes x padded nodes / 8 bytes exceeds BS_IPF_TABLE_MAX_BYTES");
  return BS_OK;
}

int host_port_check(bs_engine* e, const char* who) {
  const Refuse bad{e, who};
  if (!(e->hp.have_node && e->hp.have_pod))
    return bad(BS_E_STATE, "the PodFitsHostPorts filter needs its node and pod sides");
  if (e->hp.entries < 64 && (e->hp.want_all >> e->hp.entries))
    return bad(BS_E_INDEX, "a pod's want bit is outside the node side's host-port dictionary");
  return BS_OK;
}

// The LOC pre-pass on the main stream: each name's scaled size, then the class x node IL table.  Only after either
// side or a weight changed, and only while the ImageLocality weight is non-zero (else the table is not read).
int locality_prepass(bs_engine* e) {
  if (!e->loc.dirty || !e->w_img) return BS_OK;
  const uint32_t C = e->loc.classes, I = e->loc.images;
  if (C && e->Npad) {
    CK(e->loc.d_il.ensure((size_t)C * e->Npad));
    CK(e->loc.d_img_scaled.ensure((size_t)std::max(I, 1u) * 8));
    CK(launch_locality_prepass(e->loc.d_img_bits.as<uint32_t>(), e->loc.d_img_size.as<int64_t>(), e->loc.d_img_scaled.as<int64_t>(),
                               I, e->loc.d_off.as<uint32_t>(), e->loc.d_ids.as<uint32_t>(), e->loc.d_il.as<uint8_t>(), C,
                               e->N, e->Npad, e->s));
    e->launches += 2;
  }
  e->loc.dirty = false;
  return BS_OK;
}

// The IPA pre-pass on the main stream: M and S over the bound pods (after a node-side change), then the pod class x
// node raw table.  Only after either side changed, and only while the weight is non-zero.
int interpod_prepass(bs_engine* e) {
  if (!e->ipa.dirty || !e->w_ipa) return BS_OK;
  const uint32_t C = e->ipa.pclasses, Npad = e->Npad;
  const InterpodNodeSide& s = e->ipa.node;
  if (e->ipa.mass_dirty) {
    CK(e->ipa.d_ms.ensure((size_t)std::max<uint64_t>(s.slots, 1) * 16));
    CK(cudaMemsetAsync(e->ipa.d_ms.p, 0, (size_t)s.slots * 16, e->s));
  }
  if (C && Npad) {
    CK(e->ipa.d_raw.ensure((size_t)C * Npad * 8));
    const InterpodClasses bound{s.d_boff.as<uint32_t>(), s.d_bterm.as<uint32_t>(), s.d_bown.as<int32_t>(),
                                s.d_bmatch.as<uint8_t>(), s.bclasses};
    const InterpodClasses pods{e->ipa.d_poff.as<uint32_t>(), e->ipa.d_pterm.as<uint32_t>(), e->ipa.d_pown.as<int32_t>(),
                               e->ipa.d_pmatch.as<uint8_t>(), C};
    CK(launch_interpod_prepass(e->ipa.mass_dirty, s.d_topo.as<uint32_t>(), s.d_term_key.as<uint32_t>(),
                               s.d_term_off.as<uint32_t>(), s.d_bound_node.as<uint32_t>(), s.d_bound_class.as<uint32_t>(),
                               s.bound, bound, pods, e->ipa.d_ms.as<int64_t>(), e->ipa.d_raw.as<int64_t>(), e->N, Npad, e->s));
    e->launches += (e->ipa.mass_dirty && s.bound) ? 2 : 1;
    e->ipa.mass_dirty = false;
  }
  e->ipa.dirty = false;
  return BS_OK;
}

// The MatchInterPodAffinity filter's pre-pass on the main stream (interpod_filter.cuh): presence planes and term
// counts over the bound pods, then the class bit planes.  Only while the filter is on and after a side changed or the
// filter was switched on.
int interpod_filter_prepass(bs_engine* e) {
  if (!e->ipf.on || !e->ipf.dirty) return BS_OK;
  const uint32_t C = e->ipf.pclasses, Wg = e->Npad / 32;
  const InterpodNodeSide& s = e->ipf.node;
  const uint64_t words = (s.slots + 31) / 32;
  CK(e->ipf.d_presence.ensure((size_t)std::max<uint64_t>(2 * words, 1) * 4));
  CK(e->ipf.d_hits.ensure((size_t)std::max(s.terms, 1u) * 4));
  CK(e->ipf.d_bits.ensure((size_t)std::max<uint64_t>(3ull * C * Wg, 1) * 4));
  if (words) CK(cudaMemsetAsync(e->ipf.d_presence.p, 0, (size_t)2 * words * 4, e->s));
  if (s.terms) CK(cudaMemsetAsync(e->ipf.d_hits.p, 0, (size_t)s.terms * 4, e->s));
  const IpfTopo tp{s.d_topo.as<uint32_t>(), s.d_term_key.as<uint32_t>(), s.d_term_off.as<uint32_t>(), e->N};
  uint32_t* mbits = e->ipf.d_presence.as<uint32_t>();
  if (s.bound) {
    const IpfBound b{s.d_bound_node.as<uint32_t>(), s.d_bound_class.as<uint32_t>(), s.d_boff.as<uint32_t>(),
                     s.d_bterm.as<uint32_t>(), s.d_bown.as<int32_t>(), s.d_bmatch.as<uint8_t>(), s.bound};
    ipf_presence_kernel<<<cdiv(s.bound, IPF_THREADS), IPF_THREADS, 0, e->s>>>(b, tp, mbits, mbits + words,
                                                                         e->ipf.d_hits.as<uint32_t>());
    e->launches += 1;
  }
  const IpfPods pc{e->ipf.d_poff.as<uint32_t>(), e->ipf.d_pterm.as<uint32_t>(), e->ipf.d_prole.as<uint8_t>(),
                   e->ipf.d_pself.as<uint8_t>(), C};
  for (uint32_t c0 = 0; c0 < C && Wg; c0 += 32768) {
    const dim3 grid(cdiv(Wg * 32, IPF_THREADS), std::min(32768u, C - c0));
    ipf_class_kernel<<<grid, IPF_THREADS, 0, e->s>>>(pc, tp, mbits, mbits + words, e->ipf.d_hits.as<uint32_t>(),
                                                     e->ipf.d_bits.as<uint32_t>(), Wg, c0);
    e->launches += 1;
  }
  CK(cudaGetLastError());
  e->ipf.dirty = false;
  return BS_OK;
}

// The side tables belong to the node snapshot (the non-zero column, taints, labels, images and annotations of its
// nodes, the pods bound to them) and to the pod table: each half falls with a new table or changed rows and is
// uploaded again.
void drop_node_sides(bs_engine* e) {
  e->nz.have_node = e->pref.have_node = e->loc.have_img_node = e->loc.have_avoid_node = e->spread.have_node =
      e->ipa.have_node = e->ipf.have_node = e->hp.have_node = false;
}
void drop_pod_sides(bs_engine* e) {
  e->nz.have_pod = e->pref.have_pod = e->loc.have_img_pod = e->loc.have_avoid_pod = e->spread.have_pod =
      e->ipa.have_pod = e->ipf.have_pod = e->ipf.have_placed = e->hp.have_pod = false;
}

int evaluate_async_locked(bs_engine* e) {
  int rc;
  if (!e->have_nodes || !e->have_pods || !e->have_groups)
    return fail(e, BS_E_STATE, "bs_evaluate: upload nodes, groups and pods first");
  if ((e->out_flags & BS_OUT_PRIORITY) &&
      ((rc = nonzero_check(e, "bs_evaluate")) || (rc = preference_check(e, "bs_evaluate")) ||
       (rc = locality_check(e, "bs_evaluate")) || (rc = spread_check(e, "bs_evaluate")) ||
       (rc = interpod_check(e, "bs_evaluate"))))
    return rc;
  if (e->ipf.on && (rc = interpod_filter_check(e, "bs_evaluate"))) return rc;
  if (e->hp.on && (rc = host_port_check(e, "bs_evaluate"))) return rc;
  if (e->peer_broken)
    return fail(e, BS_E_PEER, "peer exchange is broken (a rank did not arrive): bs_peer_detach on every rank, then init/attach again");
  if (e->peer_attached && cdiv(std::max(e->G, 1u), 32) > e->peer_wpr) {
    // the push carries words_per_rank words: a round whose admits cannot all reach the peers does not run (the
    // group table is replicated, so every rank refuses the same round and none is left waiting)
    const uint32_t need = cdiv(std::max(e->G, 1u), 32);
    e->err = "bs_evaluate: the group table needs " + std::to_string(need) + " admit-bitmap words per rank, but the peer "
             "exchange carries " + std::to_string(e->peer_wpr) + " (bs_peer_init with words_per_rank >= " +
             std::to_string(need) + ")";
    return BS_E_STATE;
  }
  BS_DEVICE_GUARD(e);
  bool reprepare = e->nodes_dirty;
  if (e->classes_dirty) {
    const bool pods_changed = e->pod_classes_dirty;   // the fit classes (class_fit bits) come from the pods only
    const auto tc0 = std::chrono::steady_clock::now();
    if ((rc = rebuild_classes(e))) return rc;
    e->last_classes_us = std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - tc0).count();
    reprepare = reprepare || pods_changed;
  }
  {
    const LaneMap lm = classify_lanes(e);
    if (!e->lane_map_valid || memcmp(&lm, &e->lane_map, sizeof(lm)) != 0) {
      e->lane_map = lm;
      e->lane_map_valid = true;
      reprepare = true;
    }
  }
  if ((rc = ensure_round_buffers(e))) return rc;
  for (int k = 0; k < BS_K_COUNT; ++k) e->k_valid[k] = false;
  if (e->ipf.on && (e->ipf.dirty || e->ipf.walk_prepass)) {   // new pass bits: the class fit bits and gates are built again
    if ((rc = interpod_filter_prepass(e))) return rc;
    reprepare = true;
    e->ipf.walk_prepass = false;
  }
  if (e->hp.on && e->hp.dirty) {   // new used masks: likewise
    reprepare = true;
    e->hp.dirty = false;
  }
  if (reprepare && (rc = prepare_nodes(e))) return rc;

  const uint32_t P = e->P, G = e->G, L = e->L;
  NodeTab t = node_tab(e);
  PodTab pt = pod_tab(e);
  GroupTab gt = group_tab(e);
  GroupEff ge = group_eff(e);
  PrefixOut po = prefix_out(e);
  RoundState* st = e->d_state.as<RoundState>();

  // fork the sort stream
  CK(cudaEventRecord(e->ev_fork, e->s));
  CK(cudaStreamWaitEvent(e->s2, e->ev_fork, 0));
  CK(cudaStreamWaitEvent(e->s3, e->ev_fork, 0));
  {
    StageTimer tm(e, BS_K_SORT, e->s2);
    // one persistent kernel: group keys -> sort -> dense group rank -> pod keys -> sort -> order + rank
    e->sort_shape = {};
    e->sort_shape.valid = true;
    if (P || G) {
      SortArgs sa{};
      sa.creation = e->d_creation.as<int64_t>();
      sa.name_rank = e->d_name_rank.as<uint32_t>();
      sa.G = G;
      sa.gk0 = e->d_gk0.as<uint64_t>();
      sa.gk1 = e->d_gk1.as<uint64_t>();
      sa.group_rank = e->d_group_rank.as<uint32_t>();
      sa.prio = e->d_prio.as<int32_t>();
      sa.gid = e->d_gid.as<int32_t>();
      sa.ts = e->d_ts.as<int64_t>();
      sa.pflags = e->d_pflags.as<uint8_t>();
      sa.P = P;
      sa.pk0 = e->d_pk0.as<uint64_t>();
      sa.pk1 = e->d_pk1.as<uint64_t>();
      sa.order = e->d_order.as<uint32_t>();
      sa.rank = e->d_rank.as<uint32_t>();
      sa.idx_a = e->d_idx_a.as<uint32_t>();
      sa.idx_b = e->d_idx_b.as<uint32_t>();
      sa.hist = e->d_ghist.as<uint32_t>();
      sa.tilecnt = e->d_tilecnt.as<uint32_t>();
      sa.barrier = e->d_sort_barrier.as<unsigned int>();
      sa.ntiles_max = cdiv(std::max(std::max(P, G), 1u), SORT_TILE);
      sa.n_gpass = build_passes(e->group_stats.vary_name(), e->group_stats.vary_creation(), sa.gpass);
      // word1 = [~biased prio : 32][grouped : 1][group rank or 0x7fffffff : 31]
      const PodStats& ps = e->pod_stats;
      const uint64_t vary1 = (ps.vary_prio() << 32) | 0x80000000ull |
                             ((ps.lister_miss || ps.max_gid >= (int64_t)G) ? 0x7fffffffull : low_bits_mask(G));
      sa.n_ppass = build_passes(ps.vary_ts(), vary1, sa.ppass);
      if (std::max(P, G) <= (uint32_t)SORT_SMALL_MAX) {
        // small tables: one CTA, the same radix passes with the index arrays in shared memory
        const size_t smem = sort_small_smem();
        CK(cudaFuncSetAttribute(queue_sort_small_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        queue_sort_small_kernel<<<1, SORT_SMALL_THREADS, smem, e->s2>>>(sa);
        CK(cudaGetLastError());
        e->sort_shape.kernel = 1;
        e->sort_shape.grid = 1;
      } else {
        CK(cudaMemsetAsync(sa.barrier, 0, sizeof(unsigned int), e->s2));
        const uint32_t grid = std::max(1u, std::min(sa.ntiles_max, e->sort_max_grid));
        void* params[] = {&sa};
        // Two builds of the same kernel.  Beside a long fit kernel the sort is hidden anyway and must stay out of its
        // way (32 registers: its CTAs share their SMs with the fit CTAs); when the fit kernel is the shorter of the two
        // (a small shard, few nodes) the round waits for the sort, and the build with 16 gathers in flight per thread
        // is the faster one.  Estimate: pairs x the per-pair time of the output mode measured on an H100 (top-K: K = 16
        // at cfg4, profiles/topk_h100.jsonl; score mode on compressible memory: profiles/score_memory_h100.jsonl).
        const double score_ms = e->d_score.a.compressed() ? 2.2e-9 : 2.9e-9;
        const double per_pair_ms = (e->out_flags & BS_OUT_SCORE) ? score_ms : (e->out_flags & BS_OUT_TOPK) ? 2.0e-9 : 0.9e-9;
        const double est_fit_ms = (double)P * (double)e->N * per_pair_ms;
        const bool lean = est_fit_ms > 0.6;
        const void* fn = lean ? (const void*)queue_sort_kernel<SORT_LEAN_GROUP> : (const void*)queue_sort_kernel<SORT_WIDE_GROUP>;
        CK(cudaLaunchCooperativeKernel(fn, dim3(grid), dim3(SORT_THREADS), params, 0, e->s2));
        e->sort_shape.kernel = lean ? 2 : 3;
        e->sort_shape.grid = grid;
      }
      e->sort_shape.group_passes = sa.n_gpass;
      e->sort_shape.pod_passes = sa.n_ppass;
      tm.launched();
    }
  }
  CK(cudaEventRecord(e->ev_join, e->s2));

  // side stream (high priority): group preparation + findMaxPG, cluster scans, PreFilter.  The fit
  // kernel does not need any of it; only the per-group verdicts do, and they come after both.
  {
    StageTimer tm(e, BS_K_FIND_MAX, e->s3);
    const uint32_t gb = cdiv(std::max(G, 1u), 256);
    group_reset_kernel<<<gb, 256, 0, e->s3>>>(gt, ge, e->d_new_denied.as<uint8_t>(),
                                             e->d_admit_bitmap.as<uint32_t>(), e->d_okA.as<uint8_t>());
    tm.launched();
    if (P) {
      group_first_pod_kernel<<<cdiv(P, 256), 256, 0, e->s3>>>(pt, gt, ge);
      tm.launched();
    }
    if (G) {
      group_effective_kernel<<<gb, 256, 0, e->s3>>>(pt, gt, ge);
      tm.launched();
    }
    const uint32_t nmp = cdiv(std::max(G, 1u), FINDMAX_THREADS * FINDMAX_PER_THREAD);
    find_max_partial_kernel<<<nmp, FINDMAX_THREADS, 0, e->s3>>>(gt, ge, e->d_max_partial.as<MaxState>());
    find_max_final_kernel<<<1, 1024, 0, e->s3>>>(gt, ge, e->d_max_partial.as<MaxState>(), nmp, st, e->N);
    tm.launched(2);
  }
  // ordered cluster scans (compareClusterResourceAndRequire) per rep class
  {
    StageTimer tm(e, BS_K_CLASS_PREFIX, e->s3);
    if (e->N && G && P) {
      PrefixScratch psc = prefix_scratch(e);
      PrefixSel ps{e->d_rsel.as<uint64_t>(), e->d_rtol.as<uint64_t>(), e->d_raff.as<uint32_t>(), 0, 0, 0, 0, 0.f, st};
      for (uint32_t c0 = 0; c0 < e->n_rep_classes; c0 += e->prefix_slots) {
        const uint32_t nc = std::min(e->prefix_slots, e->n_rep_classes - c0);
        ps.c0 = c0;
        ps.mode = 0;
        launch_prefix(L, t, ps, psc, po, nc, e->s3);
        group_check_kernel<<<cdiv(G * 32, 256), 256, 0, e->s3>>>(t, gt, ge, po, c0, nc, st, e->d_okA.as<uint8_t>());
        tm.launched(3);
      }
      ps.c0 = 0;
      ps.mode = 1;
      launch_prefix(L, t, ps, psc, po, 1, e->s3);
      tm.launched(2);
    }
  }
  {
    StageTimer tm(e, BS_K_PREFILTER, e->s3);
    if (P) {
      prefilter_kernel<<<cdiv(P, PREFILTER_THREADS), PREFILTER_THREADS, 0, e->s3>>>(
          t, pt, gt, ge, po, st, e->d_okA.as<uint8_t>(), e->d_prefilter.as<uint8_t>(),
          e->d_new_denied.as<uint8_t>());
      tm.launched();
    }
    if (G) {
      group_idle_admit_kernel<<<cdiv(G, 256), 256, 0, e->s3>>>(gt, ge, e->d_admit.as<uint8_t>(),
                                                              e->d_admit_bitmap.as<uint32_t>());
      tm.launched();
    }
  }
  CK(cudaEventRecord(e->ev_pre, e->s3));
  {
    StageTimer tm(e, BS_K_GANG_FIT, e->s, true);
    if (P) {
      FitArgs a;
      a.left_w = e->d_left_w.as<int64_t>();
      a.left_n = e->d_left_n.as<int32_t>();
      a.lm = e->lane_map;
      a.left_w_pitch = (uint64_t)e->Npad * 8;
      a.left_n_pitch = (uint64_t)e->Npad * 4;
      a.classfit = e->d_classfit.as<ColBits>();
      a.req = e->d_req.as<int64_t>();
      a.req_present = e->d_ppres.as<uint32_t>();
      a.fit_class = e->d_pod_fit_class.as<uint32_t>();
      a.feasible_count = e->d_feasible.as<uint32_t>();
      a.best_node = e->d_best_node.as<int32_t>();
      a.best_score = e->d_best_score.as<int64_t>();
      a.fit_bitmap = (e->out_flags & BS_OUT_FIT_BITMAP) ? e->d_fit_bitmap.as<uint32_t>() : nullptr;
      a.score = (e->out_flags & BS_OUT_SCORE) ? e->d_score.as<int64_t>() : nullptr;
      a.score_pitch = e->score_pitch;
      a.bitmap_pitch = e->bitmap_pitch;
      a.P = P; a.N = e->N; a.Npad = e->Npad; a.W = e->W;
      a.best_packed = e->d_best_packed.as<unsigned long long>();
      const bool topk = (e->out_flags & BS_OUT_TOPK) != 0;
      a.topk_node = topk ? e->d_topk_node.as<int32_t>() : nullptr;
      a.topk_score = topk ? e->d_topk_score.as<int64_t>() : nullptr;
      a.topk_k = e->topk;
      uint32_t nl = 1;
      CK(launch_fit(a, cdiv(P, PODS_PER_CTA), e->s, &nl, e->profiling ? e->ev_a[BS_K_GANG_FIT].h : nullptr,
                    e->profiling ? e->ev_b[BS_K_GANG_FIT].h : nullptr));
      if (e->profiling) e->k_valid[BS_K_GANG_FIT] = true;
      tm.launched(nl);
    }
  }
  CK(cudaStreamWaitEvent(e->s, e->ev_pre, 0));   // PreFilter verdicts, effective group state, RoundState
  if (P && G) {
    AdmitArgs aa{};
    aa.gid = e->d_gid.as<int32_t>();
    aa.prefilter = e->d_prefilter.as<uint8_t>();
    aa.feasible_count = e->d_feasible.as<uint32_t>();
    aa.min_member = gt.min_member; aa.scheduled = gt.scheduled; aa.matched = gt.matched;
    aa.in_round = ge.in_round; aa.contrib = ge.contrib; aa.done = ge.done;
    aa.admit = e->d_admit.as<uint8_t>();
    aa.admit_bitmap = e->d_admit_bitmap.as<uint32_t>();
    aa.P = P; aa.G = G;
    gang_admit_kernel<<<cdiv(P, 256), 256, 0, e->s>>>(aa);
    e->k_launches[BS_K_GANG_FIT] += 1;
    e->launches += 1;
  }
  {
    StageTimer tm(e, BS_K_FILTER, e->s);
    if (P && (e->out_flags & BS_OUT_FILTER)) {
      FilterArgs fa;
      fa.left_plain = e->d_left_plain.as<int64_t>();
      fa.node_flags = e->d_nflags.as<uint8_t>();
      fa.req = e->d_req.as<int64_t>();
      fa.req_present = e->d_ppres.as<uint32_t>();
      fa.gid = e->d_gid.as<int32_t>();
      fa.emin_res = ge.min_res;
      fa.emin_res_present = ge.min_res_present;
      fa.eflags = ge.flags;
      fa.st = st;
      fa.filter_bitmap = e->d_filter_bitmap.as<uint32_t>();
      fa.filter_code = e->d_filter_code.as<uint8_t>();
      fa.P = P; fa.N = e->N; fa.Npad = e->Npad; fa.W = e->W; fa.G = G; fa.L = L;
      const uint32_t warps = cdiv(P, FILTER_PPW);
      filter_kernel<<<cdiv(warps * 32, 256), 256, 0, e->s>>>(fa);
      tm.launched();
    }
  }
  {
    StageTimer tm(e, BS_K_REASONS, e->s);
    if (P && (e->out_flags & BS_OUT_REASONS)) {
      ReasonHpArgs ra;
      ra.left = e->d_left_full.as<int64_t>();
      ra.left_present = e->d_left_present.as<uint32_t>();
      ra.gate = e->d_reason_gate.as<uint32_t>();
      ra.class_bins = e->d_reason_class.as<uint32_t>();
      ra.req = e->d_req.as<int64_t>();
      ra.req_present = e->d_ppres.as<uint32_t>();
      ra.fit_class = e->d_pod_fit_class.as<uint32_t>();
      ra.rows = e->d_reasons.as<uint32_t>();
      ra.P = P; ra.N = e->N; ra.Npad = e->Npad; ra.Wg = e->Npad / 32; ra.L = L;
      ra.cipf = e->ipf.d_fipf.as<uint32_t>();
      ra.ipf_bits = e->ipf.d_bits.as<uint32_t>();
      ra.n_ipf = e->ipf.pclasses;
      ra.ipf_rows = e->ipf.d_reasons.as<uint32_t>();
      ra.cconf = e->hp.d_fconf.as<uint64_t>();
      ra.hp_bins = e->hp.d_bins.as<uint32_t>();
      ra.used = e->hp.d_used.as<uint64_t>();
      ra.hp_rows = e->hp.d_reasons.as<uint32_t>();
      const uint32_t grid = cdiv(P, REASON_PODS_PER_CTA);
      with_flags<4>((e->ipf.on ? 1u : 0u) | (e->hp.on ? 2u : 0u), [&](auto f) {   // bit 0 IPF, bit 1 HP
        reason_pod_kernel<(f & 1u) != 0, (f & 2u) != 0><<<grid, REASON_THREADS, 0, e->s>>>(ra);
      });
      tm.launched();
    }
  }
  if (P && (e->out_flags & BS_OUT_PRIORITY)) {
    PriorityRatioArgs pa;
    pa.left = e->d_left_full.as<int64_t>();
    pa.left_present = e->d_left_present.as<uint32_t>();
    pa.gate = (e->ipf.on || e->hp.on) ? e->filt.d_gate.as<uint32_t>() : e->d_reason_gate.as<uint32_t>();
    pa.req = e->d_req.as<int64_t>();
    pa.req_present = e->d_ppres.as<uint32_t>();
    pa.fit_class = e->d_pod_fit_class.as<uint32_t>();
    pa.alloc = e->d_alloc.as<int64_t>();
    pa.node_nz = e->nz.d_node.as<int64_t>();
    pa.pod_nz = e->nz.d_pod.as<int64_t>();
    pa.out_node = e->d_prio_node.as<int32_t>();
    pa.out_score = e->d_prio_score.as<int64_t>();
    pa.w = e->weights;
    pa.P = P; pa.N = e->N; pa.Npad = e->Npad; pa.Wg = e->Npad / 32; pa.L = L; pa.K = e->topk;
    pa.node_requested = e->d_requested.as<int64_t>();
    pa.node_alloc_present = e->d_apres.as<uint32_t>();
    pa.node_req_present = e->d_rpres.as<uint32_t>();
    pa.ratio = e->ratio;
    const uint32_t grid = cdiv(P, PRIO_PODS_PER_CTA);
    PriorityIpaArgs la;
    static_cast<PriorityRatioArgs&>(la) = pa;
    la.prefer_taints = e->pref.d_prefer_taints.as<uint64_t>();
    la.pref_weights = e->pref.d_weights.as<int32_t>();
    la.prefer_tol = e->pref.d_prefer_tol.as<uint64_t>();
    la.pref_class = e->pref.d_class.as<uint32_t>();
    la.w_taint = e->w_taint;
    la.w_naff = e->w_naff;
    const uint32_t terms = (e->ratio.weight ? PRIO_RATIO : 0u) | (e->w_taint || e->w_naff ? PRIO_PREF : 0u) |
                           (e->w_img || e->w_avoid ? PRIO_LOC : 0u) | (e->w_spread ? PRIO_SPREAD : 0u) |
                           (e->w_ipa ? PRIO_IPA : 0u);
    if (terms & PRIO_LOC) {   // (the pre-pass runs on the same stream, ahead of the kernel)
      if ((rc = locality_prepass(e))) return rc;
      la.il = e->loc.d_il.as<uint8_t>();
      la.avoid_mask = e->loc.d_avoid_mask.as<uint64_t>();
      la.loc_class = e->loc.d_class.as<uint32_t>();
      la.avoid_bit = e->loc.d_avoid_bit.as<uint8_t>();
      la.w_img = e->w_img;
      la.w_avoid = e->w_avoid;
    }
    if (terms & PRIO_SPREAD) {
      la.spread_zone = e->spread.d_zone.as<uint8_t>();
      la.spread_counts = e->spread.d_counts.as<int32_t>();
      la.spread_class = e->spread.d_class.as<uint32_t>();
      la.w_spread = e->w_spread;
    }
    if (terms & PRIO_IPA) {   // (the pre-pass runs on the same stream, ahead of the kernel)
      if ((rc = interpod_prepass(e))) return rc;
      la.ipa_raw = e->ipa.d_raw.as<int64_t>();
      la.ipa_class = e->ipa.d_class.as<uint32_t>();
      la.w_ipa = e->w_ipa;
    }
    CK(launch_priority(L, grid, terms, la, e->s));
    e->launches += 1;
  }
  if (e->peer_attached) {
    // admit-bitmap all-gather over peer memory (kernels.cuh K8): the push is the round's last kernel on
    // the main stream, ordered behind the PREVIOUS round's wait (slot reuse rule); the wait for this
    // round's slots spins on the side stream s4 while the next round may already be computing.
    PeerArgs pa{};
    for (uint32_t r = 0; r < e->peer_world; ++r) pa.peer_buf[r] = reinterpret_cast<uint32_t*>(e->peer_ptr[r]);
    pa.local_bitmap = e->d_admit_bitmap.as<uint32_t>();
    pa.rank = e->peer_rank; pa.world = e->peer_world; pa.words_per_rank = e->peer_wpr;
    pa.n_words = std::min(e->peer_wpr, cdiv(std::max(G, 1u), 32));
    pa.seq = ++e->peer_seq;
    pa.err = e->d_peer_err.as<int>();
    pa.timeout_ns = e->peer_timeout_ns;
    if (pa.seq > 1) CK(cudaStreamWaitEvent(e->s, e->ev_gath, 0));
    {
      StageTimer tm(e, BS_K_PEER, e->s);
      peer_push_kernel<<<e->peer_world, 256, 0, e->s>>>(pa);
      tm.launched();
    }
    CK(cudaEventRecord(e->ev_push, e->s));
    CK(cudaStreamWaitEvent(e->s4, e->ev_push, 0));
    peer_wait_kernel<<<1, 32, 0, e->s4>>>(pa);
    e->k_launches[BS_K_PEER] += 1;
    e->launches += 1;
    CK(cudaEventRecord(e->ev_gath, e->s4));
  }
  CK(cudaStreamWaitEvent(e->s, e->ev_join, 0));
  CK(cudaGetLastError());
  e->ipf.round = e->ipf.on;
  e->hp.round = e->hp.on;
  e->evaluated = true;
  e->fetched = false;
  e->gang_applied = false;
  return BS_OK;
}

int fetch_locked(bs_engine* e, bs_results* out, bool view = false) {
  if (!e->evaluated) return fail(e, BS_E_STATE, "bs_fetch: nothing evaluated");
  const uint32_t P = e->P, G = e->G;
  HP_BEGIN(e);
  if (!e->fetched) {
    if (e->arena_bytes)   // every decision vector in one DMA (the arena layout is the same on both sides)
      CK(cudaMemcpyAsync(e->h_arena.p, e->d_arena.p, e->arena_bytes, cudaMemcpyDeviceToHost, e->s));
    CK(cudaStreamSynchronize(e->s));
    e->fetched = true;
  }
  HP(e, "fetch:d2h+wait");
  const RoundState* st = e->h_state.as<RoundState>();
  if (e->gang.active && e->gang.groups.size() == G && !e->gang_applied) {
    // AddToDenyCache for every group a pod of the round hit "cluster resource not enough" in (core.go:142,163)
    const uint8_t* nd = e->h_new_denied.as<uint8_t>();
    for (uint32_t g = 0; g < G; ++g)
      if (nd[g]) e->gang.deny(g, e->cycle_now_ns);
    e->gang_applied = true;
  }
  if (out && view) {
    out->prefilter = e->h_prefilter.as<uint8_t>();
    out->feasible_count = e->h_feasible.as<uint32_t>();
    out->best_node = e->h_best_node.as<int32_t>();
    out->best_score = e->h_best_score.as<int64_t>();
    out->admit = e->h_admit.as<uint8_t>();
    out->admit_bitmap = e->h_admit_bitmap.as<uint32_t>();
    out->new_denied = e->h_new_denied.as<uint8_t>();
    out->order = e->h_order.as<uint32_t>();
    out->rank = e->h_rank.as<uint32_t>();
    out->filter_code = (e->out_flags & BS_OUT_FILTER) ? e->h_filter_code.as<uint8_t>() : nullptr;
    out->max_group = st->max_group;
    out->max_finished = st->max_finished;
  } else if (out) {
    auto cp = [](void* dst, const View& src, size_t bytes) {
      if (dst && bytes) memcpy(dst, src.p, bytes);
    };
    cp(out->prefilter, e->h_prefilter, P);
    cp(out->feasible_count, e->h_feasible, (size_t)P * 4);
    cp(out->best_node, e->h_best_node, (size_t)P * 4);
    cp(out->best_score, e->h_best_score, (size_t)P * 8);
    cp(out->admit, e->h_admit, G);
    cp(out->admit_bitmap, e->h_admit_bitmap, (size_t)cdiv(G, 32) * 4);
    cp(out->new_denied, e->h_new_denied, G);
    cp(out->order, e->h_order, (size_t)P * 4);
    cp(out->rank, e->h_rank, (size_t)P * 4);
    out->max_group = st->max_group;
    out->max_finished = st->max_finished;
    if (e->out_flags & BS_OUT_FILTER) cp(out->filter_code, e->h_filter_code, P);
  }
  HP(e, "fetch:copy-out");
  if (st->ref_panic)
    return fail(e, BS_E_REF_PANIC, "findMaxPG: MinMember == 0 with Status.Scheduled != 0 (core.go:716-717 divides by zero)");
  return BS_OK;
}

// ---- preemption (preempt.cuh) ----
// What the bound-table pass finds wrong, in the order the errors are reported.
struct BoundStats {
  bool bad_index = false, bad_count = false, bad_keys = false, bad_range = false;   // bad_index: node or gid
  int32_t max_gid = -1;
  void merge(const BoundStats& o) {
    bad_index = bad_index || o.bad_index;
    bad_count = bad_count || o.bad_count;
    bad_keys = bad_keys || o.bad_keys;
    bad_range = bad_range || o.bad_range;
    max_gid = std::max(max_gid, o.max_gid);
  }
};

// preempt.cuh: the build of the preemption kernels for L lanes and the PodFitsHostPorts switch.  f(M, H) launches
// with PreemptArgsOf<H> and WalkArgsOf<H>: without the filter, the base part of PreemptHpArgs and WalkHpArgs.
template <class F>
void with_preempt_build(uint32_t L, bool hp, F&& f) {
  with_maxl<5, 9, 16>(L, [&](auto M) {
    if (hp) f(M, std::true_type{});
    else f(M, std::false_type{});
  });
}

// bs_preempt's and bs_preempt_walk's read-back: the per-preemptor columns, with the caller's other copies (more())
// before the synchronisation, the victim offsets and total (clamped to 32 bits; the walk's total is at most V, a row
// is evicted once), the victim list's checks, and the victims from a.victims, which emit(total) fills first where the
// kernels have not.
template <class More, class Emit>
int preempt_read_back(bs_engine* e, const char* who, PreemptArgs& a, uint32_t n, bs_preempt_result* out, More&& more,
                      Emit&& emit) {
  const Refuse bad{e, who};
  int rc;
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(out->node, a.out_node, (size_t)n * 4, cudaMemcpyDeviceToHost, e->s));
  CK(cudaMemcpyAsync(out->n_victims, a.out_nv, (size_t)n * 4, cudaMemcpyDeviceToHost, e->s));
  CK(cudaMemcpyAsync(out->n_candidates, a.out_cand, (size_t)n * 4, cudaMemcpyDeviceToHost, e->s));
  if ((rc = more())) return rc;
  CK(cudaStreamSynchronize(e->s));
  uint64_t total = 0;
  for (uint32_t i = 0; i < n; ++i) {
    out->victim_offset[i] = (uint32_t)std::min<uint64_t>(total, UINT32_MAX);
    total += out->n_victims[i];
  }
  out->victim_offset[n] = (uint32_t)std::min<uint64_t>(total, UINT32_MAX);
  out->victims_total = (uint32_t)std::min<uint64_t>(total, UINT32_MAX);
  if (total > out->victims_cap) return bad(BS_E_INVAL, "victims_cap is smaller than victims_total");
  if (!total) return BS_OK;
  if (!out->victims) return bad(BS_E_INVAL, "null victims buffer");
  if ((rc = emit(total))) return rc;
  CK(cudaMemcpyAsync(out->victims, a.victims, (size_t)total * 4, cudaMemcpyDeviceToHost, e->s));
  CK(cudaStreamSynchronize(e->s));
  return BS_OK;
}

}  // namespace

// ============================================================================
extern "C" {

int bs_abi_version(void) { return BS_ABI_VERSION; }

const char* bs_strerror(int err) {
  switch (err) {
    case BS_OK: return "ok";
    case BS_E_INVAL: return "invalid argument";
    case BS_E_NODEVICE: return "no CUDA device (this engine has no CPU path)";
    case BS_E_CUDA: return "CUDA runtime error";
    case BS_E_NOMEM: return "out of memory";
    case BS_E_RANGE: return "table value outside +-2^56";
    case BS_E_STATE: return "call out of order";
    case BS_E_REF_PANIC: return "reference would panic (findMaxPG divide by zero)";
    case BS_E_INDEX: return "index out of range";
    case BS_E_PEER: return "peer exchange timed out";
  }
  return "unknown error";
}

const char* bs_last_error(const bs_engine* e) { return e ? e->err.c_str() : ""; }

int bs_create(const bs_config* cfg, bs_engine** out) {
  if (!cfg || !out) return BS_E_INVAL;
  *out = nullptr;
  if (cfg->n_lanes < BS_FIXED_LANES || cfg->n_lanes > BS_MAX_LANES) return BS_E_INVAL;
  // top-K lists: 1..BS_TOPK_MAX entries with the flag, none without; the score matrix already holds them
  // (the priority lists share K; they combine with every flag)
  if ((cfg->out_flags & (BS_OUT_TOPK | BS_OUT_PRIORITY))
          ? (cfg->topk < 1 || cfg->topk > BS_TOPK_MAX || ((cfg->out_flags & BS_OUT_TOPK) && (cfg->out_flags & BS_OUT_SCORE)))
          : cfg->topk != 0)
    return BS_E_INVAL;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) {
    cudaGetLastError();
    return BS_E_NODEVICE;
  }
  if (cfg->device < 0 || cfg->device >= ndev) return BS_E_INVAL;
  DeviceGuard guard(cfg->device);
  if (guard.err != cudaSuccess) return BS_E_CUDA;
  bs_engine* e = new (std::nothrow) bs_engine();
  if (!e) return BS_E_NOMEM;
  e->device = cfg->device;
  e->L = cfg->n_lanes;
  e->out_flags = cfg->out_flags;
  e->topk = cfg->topk;
  e->host_prof = getenv("BS_HOST_PROFILE") != nullptr;
  int prio_lo = 0, prio_hi = 0;
  cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);   // the small kernels of the PreFilter chain must get the
                                                          // SM slots the fit kernel's retiring CTAs free
  bool ok = cudaStreamCreateWithFlags(&e->s.h, cudaStreamNonBlocking) == cudaSuccess &&
            cudaStreamCreateWithFlags(&e->s2.h, cudaStreamNonBlocking) == cudaSuccess &&
            cudaStreamCreateWithPriority(&e->s3.h, cudaStreamNonBlocking, prio_hi) == cudaSuccess &&
            cudaStreamCreateWithPriority(&e->s4.h, cudaStreamNonBlocking, prio_hi) == cudaSuccess &&
            cudaEventCreateWithFlags(&e->ev_pre.h, cudaEventDisableTiming) == cudaSuccess &&
            cudaEventCreateWithFlags(&e->ev_push.h, cudaEventDisableTiming) == cudaSuccess &&
            cudaEventCreateWithFlags(&e->ev_gath.h, cudaEventDisableTiming) == cudaSuccess &&
            cudaEventCreateWithFlags(&e->ev_fork.h, cudaEventDisableTiming) == cudaSuccess &&
            cudaEventCreateWithFlags(&e->ev_join.h, cudaEventDisableTiming) == cudaSuccess &&
            cudaEventCreateWithFlags(&e->ev_classes.h, cudaEventDisableTiming) == cudaSuccess;
  for (int k = 0; ok && k < BS_K_COUNT; ++k)
    ok = cudaEventCreate(&e->ev_a[k].h) == cudaSuccess && cudaEventCreate(&e->ev_b[k].h) == cudaSuccess;
  if (ok) {
    int per_sm = 0, sms = 0;
    int per_sm_wide = 0;
    ok = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, queue_sort_kernel<SORT_LEAN_GROUP>, SORT_THREADS, 0) == cudaSuccess &&
         cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm_wide, queue_sort_kernel<SORT_WIDE_GROUP>, SORT_THREADS, 0) == cudaSuccess &&
         cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, cfg->device) == cudaSuccess;
    // the sort shares the GPU with the fit kernel on the other stream: one CTA per SM is plenty
    per_sm = std::min(per_sm, per_sm_wide);
    e->sort_max_grid = (uint32_t)std::max(1, std::min(per_sm * sms, sms));
  }
  if (!ok) {
    bs_destroy(e);
    return BS_E_CUDA;
  }
  *out = e;
  return BS_OK;
}

void bs_destroy(bs_engine* e) {
  if (!e) return;
  DeviceGuard guard(e->device);
  if (e->s) cudaStreamSynchronize(e->s);
  if (e->s2) cudaStreamSynchronize(e->s2);
  if (e->s4) cudaStreamSynchronize(e->s4);
  for (uint32_t r = 0; r < e->peer_world; ++r)
    if (r != e->peer_rank && e->peer_ptr[r]) cudaIpcCloseMemHandle(e->peer_ptr[r]);
  delete e;   // the members free their buffers, streams and events on the engine's device (the guard is still alive)
}

int bs_upload_nodes(bs_engine* e, const bs_node_table* t) {
  if (!e || !t) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  drop_node_sides(e);
  if (t->n_lanes != e->L) return fail(e, BS_E_INVAL, "bs_upload_nodes: n_lanes differs from the engine's");
  const uint32_t N = t->n_nodes, L = e->L;
  const auto cols = node_cols(e, t);
  if (N && null_column(cols)) return fail(e, BS_E_INVAL, "bs_upload_nodes: null column");
  // the old table goes before validation and the DMA, with what belongs to it: a table that fails either (BS_E_RANGE,
  // or an error partway through the copy) leaves no snapshot behind, and the engine answers BS_E_STATE until a valid
  // one arrives instead of evaluating the previous snapshot (or a half-written one)
  e->have_nodes = false;
  e->have_bound = e->hp.have_bound = false;   // the bound-pod table belongs to the node snapshot
  if (e->n_aff) e->classes_dirty = true;   // class ids are validated again: the affinity table belongs to the
  e->n_aff = 0;                            // node snapshot and goes with it
  e->evaluated = false;
  HP_BEGIN(e);
  const NodeStats ns = node_host_pass(t, L, N);
  if (ns.bad_range) return fail(e, BS_E_RANGE, "bs_upload_nodes: value outside +-2^56");
  HP(e, "nodes:host-pass");
  BS_DEVICE_GUARD(e);
  const uint32_t Npad = std::max(1u, cdiv(N, NODE_TILE)) * NODE_TILE;
  int rc;
  if ((rc = upload_cols(e, cols, N, Npad))) return rc;
  HP(e, "nodes:dma-enqueue");
  CK(cudaStreamSynchronize(e->s));
  HP(e, "nodes:dma-wait");
  e->h_nflags.assign(t->flags, t->flags + N);
  e->h_npc.assign(t->pod_count, t->pod_count + N);
  e->h_nrpres.assign(t->req_present, t->req_present + N);
  e->node_stats = ns;
  e->N = N;
  e->score_pitch = (N + 1u) & ~1u;
  e->bitmap_pitch = (cdiv(N, 32) + 31u) & ~31u;
  e->Npad = Npad;
  e->W = cdiv(N, 32);
  e->have_nodes = true;
  e->nodes_dirty = true;
  e->evaluated = false;
  return BS_OK;
}

int bs_update_nodes(bs_engine* e, const uint32_t* idx, const bs_node_table* t) {
  if (!e || !t || (t->n_nodes && !idx)) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->have_nodes) return fail(e, BS_E_STATE, "bs_update_nodes: upload nodes first");
  drop_node_sides(e);   // the changed rows come with new side columns
  if (t->n_lanes != e->L) return fail(e, BS_E_INVAL, "bs_update_nodes: n_lanes differs from the engine's");
  const uint32_t n = t->n_nodes, L = e->L;
  if (!n) return BS_OK;
  const auto cols = node_cols(e, t);
  if (null_column(cols)) return fail(e, BS_E_INVAL, "bs_update_nodes: null column");
  for (uint32_t k = 0; k < n; ++k)
    if (idx[k] >= e->N) return BS_E_INDEX;
  const NodeStats ns = node_host_pass(t, L, n);
  if (ns.bad_range) return fail(e, BS_E_RANGE, "bs_update_nodes: value outside +-2^56");
  BS_DEVICE_GUARD(e);
  HP_BEGIN(e);
  int rc;
  if ((rc = scatter_rows(e, cols, idx, n, e->Npad))) return rc;
  HP(e, "upd-nodes:enqueue");
  CK(cudaStreamSynchronize(e->s));
  HP(e, "upd-nodes:wait");
  e->node_stats.merge(ns);
  for (uint32_t k = 0; k < n; ++k) {
    e->h_nflags[idx[k]] = t->flags[k];
    e->h_npc[idx[k]] = t->pod_count[k];
    e->h_nrpres[idx[k]] = t->req_present[k];
  }
  e->have_bound = e->hp.have_bound = false;
  e->nodes_dirty = true;
  e->evaluated = false;
  return BS_OK;
}

int bs_upload_groups(bs_engine* e, const bs_group_table* t) {
  if (!e || !t) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  if (t->n_lanes != e->L) return fail(e, BS_E_INVAL, "bs_upload_groups: n_lanes differs from the engine's");
  const uint32_t G = t->n_groups, L = e->L;
  const auto cols = group_cols(e, t);
  if (G && (null_column(cols) || !t->rep_sel || !t->rep_tol)) return fail(e, BS_E_INVAL, "bs_upload_groups: null column");
  // the DMAs go first (asynchronous from pinned tables) and run under the host checks below; a table
  // that then fails validation is dropped (have_groups = false)
  BS_DEVICE_GUARD(e);
  HP_BEGIN(e);
  e->have_groups = false;
  e->have_bound = e->hp.have_bound = false;   // the bound rows' group indices refer to the old table
  e->evaluated = false;
  const uint32_t Gp = std::max(G, 1u);
  int rc;
  if ((rc = upload_cols(e, cols, G, Gp))) return rc;
  HP(e, "groups:dma-enqueue");
  // the representative columns are compared with the engine's when it has ids assigned for a table of this length
  const bool cmp_reps = e->h_gsel.size() == G && e->h_gtol.size() == G && e->h_grc.size() == G && e->h_gaff.size() == G;
  const GroupStats gs = group_host_pass(t, L, G, cmp_reps ? e : nullptr);
  if (gs.bad_range) {
    cudaStreamSynchronize(e->s);
    return fail(e, BS_E_RANGE, "bs_upload_groups: value outside +-2^56");
  }
  if (gs.bad_creation) {
    cudaStreamSynchronize(e->s);
    return fail(e, BS_E_RANGE, "bs_upload_groups: creation_ns == INT64_MAX");
  }
  e->group_stats = gs;
  // representative (sel, tol, affinity) columns unchanged since the ids were assigned: nothing to look up again
  if (!cmp_reps || gs.reps_differ) {
    e->h_gsel.assign(t->rep_sel, t->rep_sel + G);
    e->h_gtol.assign(t->rep_tol, t->rep_tol + G);
    e->h_gaff.resize(G);
    for (uint32_t g = 0; g < G; ++g) e->h_gaff[g] = t->rep_aff_class ? t->rep_aff_class[g] : BS_AFF_NONE;
    e->group_classes_dirty = true;
    e->classes_dirty = true;
  }
  if (e->h_wait_ns.size() != G) e->h_wait_ns.assign(G, -1);
  HP(e, "groups:host-pass");
  CK(cudaStreamSynchronize(e->s));   // the caller's arrays are free again once we return
  HP(e, "groups:dma-wait");
  e->h_min_member.assign(t->min_member, t->min_member + G);
  e->h_scheduled.assign(t->scheduled, t->scheduled + G);
  e->h_matched_up.assign(t->matched, t->matched + G);
  e->h_gflags_up.assign(t->flags, t->flags + G);
  HP(e, "groups:host-copies");
  e->G = G;
  e->have_groups = true;
  e->evaluated = false;
  return BS_OK;
}

int bs_update_groups(bs_engine* e, const uint32_t* idx, const bs_group_table* t) {
  if (!e || !t || (t->n_groups && !idx)) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->have_groups) return fail(e, BS_E_STATE, "bs_update_groups: upload groups first");
  if (t->n_lanes != e->L) return fail(e, BS_E_INVAL, "bs_update_groups: n_lanes differs from the engine's");
  const uint32_t n = t->n_groups, L = e->L, G = e->G;
  if (!n) return BS_OK;
  const auto cols = group_cols(e, t);
  if (null_column(cols) || !t->rep_sel || !t->rep_tol) return fail(e, BS_E_INVAL, "bs_update_groups: null column");
  for (uint32_t k = 0; k < n; ++k)
    if (idx[k] >= G) return BS_E_INDEX;
  const GroupStats gs = group_host_pass(t, L, n, nullptr);
  if (gs.bad_range) return fail(e, BS_E_RANGE, "bs_update_groups: value outside +-2^56");
  if (gs.bad_creation) return fail(e, BS_E_RANGE, "bs_update_groups: creation_ns == INT64_MAX");
  BS_DEVICE_GUARD(e);
  HP_BEGIN(e);
  int rc;
  if ((rc = scatter_rows(e, cols, idx, n, std::max(G, 1u)))) return rc;
  HP(e, "upd-groups:enqueue");
  CK(cudaStreamSynchronize(e->s));
  HP(e, "upd-groups:wait");
  e->group_stats.merge(gs);
  for (uint32_t k = 0; k < n; ++k) {
    e->h_gsel[idx[k]] = t->rep_sel[k];
    e->h_gtol[idx[k]] = t->rep_tol[k];
    e->h_gaff[idx[k]] = t->rep_aff_class ? t->rep_aff_class[k] : BS_AFF_NONE;
    e->h_min_member[idx[k]] = t->min_member[k];
    e->h_scheduled[idx[k]] = t->scheduled[k];
    e->h_matched_up[idx[k]] = t->matched[k];
    e->h_gflags_up[idx[k]] = t->flags[k];
  }
  e->classes_dirty = true;         // the class tables go to the device again (new classes may have appeared); the pods' ids stay
  if (!e->group_classes_dirty && e->h_grc.size() == G) {
    // the other groups' ids are current: look up only the changed rows (the index keeps ids stable)
    CK(cudaEventSynchronize(e->ev_classes));   // no DMA is reading h_grc
    for (uint32_t k = 0; k < n; ++k)
      e->h_grc[idx[k]] = e->rep_index.get_or_add(ClassKey{e->h_gsel[idx[k]], e->h_gtol[idx[k]], 0u, e->h_gaff[idx[k]]});
    e->group_ids_dirty = true;
  } else {
    e->group_classes_dirty = true;
  }
  e->evaluated = false;
  return BS_OK;
}

int bs_upload_pods(bs_engine* e, const bs_pod_table* t) {
  if (!e || !t) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  drop_pod_sides(e);
  if (t->n_lanes != e->L) return fail(e, BS_E_INVAL, "bs_upload_pods: n_lanes differs from the engine's");
  const uint32_t P = t->n_pods, L = e->L;
  if (P && (!t->req || !t->req_present || !t->gid || !t->sel_mask || !t->tol_mask || !t->priority ||
            !t->ts_ns || !t->flags))
    return fail(e, BS_E_INVAL, "bs_upload_pods: null column");
  // Only now does the new table replace the old one: a call refused above keeps the old table, whose h_pfc may hold
  // the classes the filters gave it, and h_pfc_base its base classes.
  e->filt.pfc_base_valid = false;   // the new table's fit classes are its base classes
  e->filt.assign_dirty = false;
  // ONE parallel pass over the table before anything is committed: per-lane maxima (range check and
  // wide/narrow lane classification), the varying bits of the sort keys, thread-local class indices
  // (fit class = (sel, tol, scalar keys requested with a non-zero amount, core.go:688-690);
  // representative class = (sel, tol)), and the host copies the per-call mirrors read.
  const Chunks ch(P, 8192);
  std::vector<ClassIndex> fit_local(ch.T), rep_local(ch.T);
  HP_BEGIN(e);
  e->h_gid.resize(P); e->h_prio.resize(P); e->h_pflags.resize(P);
  BS_DEVICE_GUARD(e);
  CK(cudaEventSynchronize(e->ev_classes));   // the class ids of the previous table are no longer being read
  if (!e->h_pfc.resize(P) || !e->h_prc.resize(P)) return fail(e, BS_E_NOMEM, "pinned host memory");
  // the DMAs go first (asynchronous from pinned tables) and run under the host pass below; a table
  // that then fails validation is dropped (have_pods = false)
  e->have_pods = false;
  e->evaluated = false;
  const uint32_t Pp = std::max(P, 1u);
  int rc;
  if ((rc = upload_col(e, col(t->req, e->d_req, L), P, Pp))) return rc;
  if ((rc = upload_vec(e, e->d_ppres, t->req_present, P, Pp))) return rc;
  if ((rc = upload_vec(e, e->d_gid, t->gid, P, Pp))) return rc;
  if ((rc = upload_vec(e, e->d_prio, t->priority, P, Pp))) return rc;
  if ((rc = upload_vec(e, e->d_ts, t->ts_ns, P, Pp))) return rc;
  if ((rc = upload_vec(e, e->d_pflags, t->flags, P, Pp))) return rc;
  HP(e, "pods:dma-enqueue");
  const PodStats ps = ch.reduce<PodStats>([&](int tk, uint32_t a0, uint32_t a1, PodStats& st) {
    for (uint32_t d = 0; d < L; ++d) {
      const int64_t* row = t->req + (size_t)d * P;
      int64_t lo = 0, hi = 0;
      uint64_t o = 0;
      for (uint32_t p = a0; p < a1; ++p) { lo = std::min(lo, row[p]); hi = std::max(hi, row[p]); o |= (uint64_t)row[p]; }
      const int64_t neg = lo == INT64_MIN ? INT64_MAX : -lo;
      st.bad_range = st.bad_range || lo < -BS_VALUE_LIMIT || hi > BS_VALUE_LIMIT;
      st.max_req[d] = std::max(hi, neg); st.neg_req[d] = neg; st.or_req[d] = o;
    }
    {
      // reductions in locals and the plain column copies as memcpy: a byte store inside the loop would make the
      // compiler spill every accumulator (char stores alias everything)
      uint64_t ot = 0, at = ~0ull;
      uint32_t op = 0, apr = ~0u;
      int miss = 0;
      int32_t mg = -1;
      for (uint32_t p = a0; p < a1; ++p) {
        const uint64_t ts = (uint64_t)t->ts_ns[p];
        const uint32_t pr = (uint32_t)t->priority[p];
        const int32_t g = t->gid[p];
        ot |= ts; at &= ts; op |= pr; apr &= pr;
        miss |= ((g < BS_GID_NONE) || (t->flags[p] & BS_POD_LISTER_MISS)) ? 1 : 0;
        mg = std::max(mg, g);
      }
      st.or_ts = ot; st.and_ts = at; st.or_prio = op; st.and_prio = apr; st.lister_miss = miss != 0; st.max_gid = mg;
      if (a1 > a0) {
        memcpy(e->h_gid.data() + a0, t->gid + a0, (size_t)(a1 - a0) * 4);
        memcpy(e->h_prio.data() + a0, t->priority + a0, (size_t)(a1 - a0) * 4);
        memcpy(e->h_pflags.data() + a0, t->flags + a0, (size_t)(a1 - a0));
      }
    }
    {
      // one index lookup per pod: the representative class of a fit class is looked up once per class
      ClassIndex fit, rep;
      fit.clear();
      rep.clear();
      std::vector<uint32_t> rep_of_fit;
      uint32_t* pfc = e->h_pfc.data();
      uint32_t* prc = e->h_prc.data();
      for (uint32_t p = a0; p < a1; ++p) {
        uint32_t nz = 0;
        const uint32_t rp = t->req_present[p];
        for (uint32_t d = 4; d < L; ++d)
          if (((rp >> d) & 1u) && t->req[(size_t)d * P + p] != 0) nz |= 1u << d;
        const uint32_t af = t->aff_class ? t->aff_class[p] : BS_AFF_NONE;
        const uint32_t fc = fit.get_or_add(ClassKey{t->sel_mask[p], t->tol_mask[p], nz, af});
        if (fc >= rep_of_fit.size()) rep_of_fit.push_back(rep.get_or_add(ClassKey{t->sel_mask[p], t->tol_mask[p], 0u, af}));
        pfc[p] = fc;
        prc[p] = rep_of_fit[fc];
      }
      fit_local[tk] = std::move(fit);
      rep_local[tk] = std::move(rep);
    }
  });
  HP(e, "pods:host-pass");
  if (ps.bad_range) {   // the device and host-side columns were already overwritten: the table stays dropped
    cudaStreamSynchronize(e->s);
    return fail(e, BS_E_RANGE, "bs_upload_pods: value outside +-2^56");
  }
  // Merge the thread-local class indices into the engine's and remap the ids while the DMA is in
  // flight.  The engine's indices persist across uploads (ids of known classes are stable, so the
  // groups' representative ids stay valid); they restart only when mostly stale.
  {
    size_t lf = 0, lr = 0;
    for (int k = 0; k < ch.T; ++k) { lf += fit_local[k].size(); lr += rep_local[k].size(); }
    if (e->fit_index.size() > std::max<size_t>(4096, 4 * lf)) e->fit_index.clear();
    if (e->rep_index.size() > std::max<size_t>(4096, 4 * lr)) {
      e->rep_index.clear();
      e->group_classes_dirty = true;   // the groups' ids referred to the old index
    }
  }
  merge_classes(e->fit_index, fit_local, ch, e->h_pfc.data());
  merge_classes(e->rep_index, rep_local, ch, e->h_prc.data());
  HP(e, "pods:class-merge");
  CK(cudaStreamSynchronize(e->s));
  HP(e, "pods:dma-wait");
  e->pod_stats = ps;
  e->P = P;
  e->have_pods = true;
  e->classes_dirty = true;
  e->pod_classes_dirty = true;
  e->evaluated = false;
  return BS_OK;
}

int bs_upload_affinity(bs_engine* e, uint32_t n_classes, const uint32_t* bits) {
  if (!e || (n_classes && !bits)) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->have_nodes) return fail(e, BS_E_STATE, "bs_upload_affinity: upload nodes first");
  BS_DEVICE_GUARD(e);
  const size_t words = (size_t)n_classes * e->W;
  if (words) {
    CK(e->d_aff_bits.ensure(words * 4));
    CK(cudaMemcpyAsync(e->d_aff_bits.p, bits, words * 4, cudaMemcpyHostToDevice, e->s));
    CK(cudaStreamSynchronize(e->s));
  }
  e->n_aff = n_classes;
  e->nodes_dirty = true;     // class-fit bits and cluster scans follow the table
  e->classes_dirty = true;   // class ids are validated against it
  e->evaluated = false;
  return BS_OK;
}

// ---- gang state: the TTL tables around Permit as engine state (gang_state.hpp) ----
int bs_state_reset(bs_engine* e) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->have_groups) return fail(e, BS_E_STATE, "bs_state_reset: upload groups first");
  e->gang.reset(e->G);
  return BS_OK;
}

int bs_state_remap(bs_engine* e, uint32_t n_groups, const int32_t* old_index) {
  if (!e || (n_groups && !old_index)) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  e->gang.remap(n_groups, old_index);
  return BS_OK;
}

int bs_state_view(bs_engine* e, int64_t now_ns, uint32_t n_groups, uint32_t* matched, uint8_t* flags) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->gang.active || e->gang.groups.size() != n_groups) return fail(e, BS_E_STATE, "bs_state_view: tables of another shape");
  for (uint32_t g = 0; g < n_groups; ++g) {
    if (matched) matched[g] = e->gang.matched_count(g, now_ns);
    if (flags) flags[g] = (uint8_t)((e->gang.groups[g].scheduled ? BS_GROUP_SCHEDULED : 0u) | (e->gang.denied(g, now_ns) ? BS_GROUP_DENIED : 0u));
  }
  return BS_OK;
}

int bs_permitted_view(bs_engine* e, int64_t now_ns, const uint64_t* uids, uint32_t n, uint8_t* out) {
  if (!e || (n && (!uids || !out))) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  for (uint32_t i = 0; i < n; ++i) out[i] = e->gang.active && e->gang.permitted_recently(uids[i], now_ns) ? 1 : 0;
  return BS_OK;
}

int bs_state_move(bs_engine* dst, bs_engine* src) {
  if (!dst || !src || dst == src) return BS_E_INVAL;
  std::lock_guard<std::mutex> l1(src->mu);
  std::lock_guard<std::mutex> l2(dst->mu);
  dst->gang = std::move(src->gang);
  src->gang = GangState();
  return BS_OK;
}

int bs_set_pod_ids(bs_engine* e, const uint64_t* uid, const uint64_t* name_id) {
  if (!e || !uid || !name_id) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->have_pods) return fail(e, BS_E_STATE, "bs_set_pod_ids: upload pods first");
  e->h_pod_uid.assign(uid, uid + e->P);
  e->h_pod_name.assign(name_id, name_id + e->P);
  return BS_OK;
}

int bs_begin_cycle(bs_engine* e, int64_t now_ns) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->have_groups || !e->have_pods) return fail(e, BS_E_STATE, "bs_begin_cycle: upload groups and pods first");
  if (!e->gang.active || e->gang.groups.size() != e->G) return fail(e, BS_E_STATE, "bs_begin_cycle: bs_state_reset after the group table changed size");
  BS_DEVICE_GUARD(e);
  const uint32_t G = e->G, P = e->P;
  e->cycle_now_ns = now_ns;
  // the go-cache views at `now` become the columns the round reads: len(MatchedPodNodes.Items()), pgs.Scheduled,
  // lastDeniedPG and lastPermittedPod membership (core.go:95-110,706,711)
  std::vector<uint32_t> matched(G);
  std::vector<uint8_t> gfl(G), pfl(P);
  for (uint32_t g = 0; g < G; ++g) {
    matched[g] = e->gang.matched_count(g, now_ns);
    uint8_t f = e->h_gflags_up[g] & ~(uint8_t)(BS_GROUP_SCHEDULED | BS_GROUP_DENIED);
    if (e->gang.groups[g].scheduled) f |= BS_GROUP_SCHEDULED;
    if (e->gang.denied(g, now_ns)) f |= BS_GROUP_DENIED;
    gfl[g] = f;
  }
  const bool ids = e->h_pod_uid.size() == P && !e->gang.permitted.empty();   // an empty lastPermittedPod: no lookups
  for (uint32_t p = 0; p < P; ++p) {
    uint8_t f = e->h_pflags[p] & ~(uint8_t)BS_POD_PERMITTED_RECENTLY;
    if (ids && e->gang.permitted_recently(e->h_pod_uid[p], now_ns)) f |= BS_POD_PERMITTED_RECENTLY;
    pfl[p] = f;
  }
  if (G) {
    CK(cudaMemcpyAsync(e->d_matched.p, matched.data(), (size_t)G * 4, cudaMemcpyHostToDevice, e->s));
    CK(cudaMemcpyAsync(e->d_gflags.p, gfl.data(), G, cudaMemcpyHostToDevice, e->s));
  }
  if (P) CK(cudaMemcpyAsync(e->d_pflags.p, pfl.data(), P, cudaMemcpyHostToDevice, e->s));
  CK(cudaStreamSynchronize(e->s));
  e->evaluated = false;
  return BS_OK;
}

int bs_permit_at(bs_engine* e, uint32_t pod, uint32_t node, int64_t now_ns, bs_permit_result* r) {
  if (!e || !r) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->have_pods || !e->have_groups) return fail(e, BS_E_STATE, "bs_permit_at: upload groups and pods first");
  if (pod >= e->P || (e->have_nodes && node >= e->N)) return BS_E_INDEX;
  const int64_t kSecond = 1000000000ll, kDefaultWait = 60 * kSecond;  // util.DefaultWaitTime k8s.go:31
  const int32_t g = e->h_gid[pod];
  memset(r, 0, sizeof(*r));
  r->group = -1;
  if (g == BS_GID_NONE) {  // core.go:270-272 + batchscheduler.go:190-193
    r->ready = 1; r->code = BS_CODE_SUCCESS; r->wait_ns = 0;
    return BS_OK;
  }
  if (g < 0 || (uint32_t)g >= e->G) {  // core.go:275-277 + batchscheduler.go:194-195
    r->ready = 0; r->code = BS_CODE_UNSCHEDULABLE; r->wait_ns = kDefaultWait;
    return BS_OK;
  }
  if (!e->gang.active || e->gang.groups.size() != e->G || e->h_pod_uid.size() != e->P)
    return fail(e, BS_E_STATE, "bs_permit_at: bs_state_reset and bs_set_pod_ids first");
  r->group = g;
  int64_t wait = e->default_wait_ns;   // util.GetWaitTimeDuration (k8s.go:82-91)
  if ((size_t)g < e->h_wait_ns.size() && e->h_wait_ns[g] >= 0) wait = e->h_wait_ns[g];
  const bool ready = e->gang.permit((uint32_t)g, e->h_pod_uid[pod], e->h_pod_name[pod], node, now_ns, wait,
                                    e->h_min_member[g], e->h_scheduled[g]);   // core.go:283-307
  r->wait_ns = wait + kSecond;           // batchscheduler.go:180-182
  r->ready = ready ? 1 : 0;
  r->start_signal = r->ready;            // :197-199
  r->code = BS_CODE_WAIT;                // :184-187 and :201
  return BS_OK;
}

int bs_expire(bs_engine* e, int64_t now_ns, uint32_t* rej_group, uint64_t* rej_uid, uint32_t rej_cap, uint32_t* n_rejected,
              uint32_t* evicted_group, uint32_t evict_cap, uint32_t* n_evicted) {
  if (!e || !n_rejected || !n_evicted) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->gang.active) return fail(e, BS_E_STATE, "bs_expire: bs_state_reset first");
  std::vector<uint32_t> rg, ev;
  std::vector<uint64_t> ru;
  e->gang.expire(now_ns, &rg, &ru, &ev);
  *n_rejected = (uint32_t)rg.size();
  *n_evicted = (uint32_t)ev.size();
  for (uint32_t i = 0; i < rg.size() && i < rej_cap; ++i) {
    if (rej_group) rej_group[i] = rg[i];
    if (rej_uid) rej_uid[i] = ru[i];
  }
  for (uint32_t i = 0; i < ev.size() && i < evict_cap; ++i)
    if (evicted_group) evicted_group[i] = ev[i];
  return BS_OK;
}

int bs_allow_list(bs_engine* e, uint32_t group, int64_t now_ns, uint64_t* uids, uint32_t* nodes, uint32_t cap, uint32_t* n) {
  if (!e || !n) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->gang.active || e->gang.groups.size() != e->G) return fail(e, BS_E_STATE, "bs_allow_list: bs_state_reset first");
  if (group >= e->G) return BS_E_INDEX;
  std::vector<uint64_t> u;
  std::vector<uint32_t> nd;
  e->gang.allow_list(group, now_ns, e->h_min_member[group], e->h_scheduled[group], &u, &nd);
  *n = (uint32_t)u.size();
  for (uint32_t i = 0; i < u.size() && i < cap; ++i) {
    if (uids) uids[i] = u[i];
    if (nodes) nodes[i] = nd[i];
  }
  return BS_OK;
}

int bs_deny(bs_engine* e, uint32_t group, int64_t now_ns) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->gang.active || e->gang.groups.size() != e->G) return fail(e, BS_E_STATE, "bs_deny: bs_state_reset first");
  if (group >= e->G) return BS_E_INDEX;
  e->gang.deny(group, now_ns);
  return BS_OK;
}

int bs_mark_permitted(bs_engine* e, uint64_t uid, int64_t now_ns) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->gang.active) return fail(e, BS_E_STATE, "bs_mark_permitted: bs_state_reset first");
  e->gang.mark_permitted(uid, now_ns);
  return BS_OK;
}

int bs_group_state(bs_engine* e, uint32_t group, int64_t now_ns, uint32_t* matched, int32_t* scheduled_flag, int32_t* denied) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->gang.active || e->gang.groups.size() != e->G) return fail(e, BS_E_STATE, "bs_group_state: bs_state_reset first");
  if (group >= e->G) return BS_E_INDEX;
  if (matched) *matched = e->gang.matched_count(group, now_ns);
  if (scheduled_flag) *scheduled_flag = e->gang.groups[group].scheduled ? 1 : 0;
  if (denied) *denied = e->gang.denied(group, now_ns) ? 1 : 0;
  return BS_OK;
}

int bs_set_wait_time(bs_engine* e, int64_t default_ns, const int64_t* per_group_ns, uint32_t n_groups) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  e->default_wait_ns = default_ns;
  if (per_group_ns) e->h_wait_ns.assign(per_group_ns, per_group_ns + n_groups);
  return BS_OK;
}

int bs_evaluate_async(bs_engine* e) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  return evaluate_async_locked(e);
}

// checks the sticky error word of the peer exchange; on a timeout the exchange is marked broken
static int peer_check_locked(bs_engine* e) {
  if (!e->peer_attached) return BS_OK;
  CK(cudaStreamSynchronize(e->s4));
  int bad = 0;
  CK(cudaMemcpy(&bad, e->d_peer_err.p, sizeof(int), cudaMemcpyDeviceToHost));
  if (bad) {
    e->peer_broken = true;
    return fail(e, BS_E_PEER, "peer exchange timed out: a rank did not arrive (detach and re-attach every rank)");
  }
  return BS_OK;
}

int bs_sync(bs_engine* e) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  BS_DEVICE_GUARD(e);
  CK(cudaStreamSynchronize(e->s));
  return peer_check_locked(e);
}

int bs_fetch(bs_engine* e, bs_results* out) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  BS_DEVICE_GUARD(e);
  return fetch_locked(e, out);
}

int bs_fetch_view(bs_engine* e, bs_results* out) {
  if (!e || !out) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  BS_DEVICE_GUARD(e);
  return fetch_locked(e, out, true);
}

int bs_evaluate_view(bs_engine* e, bs_results* out) {
  if (!e || !out) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  int rc = evaluate_async_locked(e);
  if (rc) return rc;
  BS_DEVICE_GUARD(e);
  return fetch_locked(e, out, true);
}

int bs_evaluate(bs_engine* e, bs_results* out) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  static const bool prof = getenv("BS_HOST_PROFILE") != nullptr;   // host-side stage times on stderr
  const auto t0 = std::chrono::steady_clock::now();
  int rc = evaluate_async_locked(e);
  if (rc) return rc;
  if (!prof) return fetch_locked(e, out);
  const auto t1 = std::chrono::steady_clock::now();
  {
    BS_DEVICE_GUARD(e);
    CK(cudaStreamSynchronize(e->s));
  }
  const auto t2 = std::chrono::steady_clock::now();
  rc = fetch_locked(e, out);
  const auto t3 = std::chrono::steady_clock::now();
  auto us = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b) {
    return std::chrono::duration<double, std::micro>(b - a).count();
  };
  fprintf(stderr, "[bs_evaluate] enqueue %.0f us (classes %.0f us)  device wait %.0f us  fetch %.0f us |", us(t0, t1),
          e->last_classes_us, us(t1, t2), us(t2, t3));
  for (auto& kv : e->hp_log) fprintf(stderr, " %s %.0f", kv.first, kv.second);
  fprintf(stderr, "\n");
  e->hp_log.clear();
  return rc;
}

int bs_prefilter(bs_engine* e, uint32_t pod, bs_status* st) {
  if (!e || !st) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->evaluated) return fail(e, BS_E_STATE, "bs_prefilter: evaluate first");
  if (pod >= e->P) return BS_E_INDEX;
  if (!e->fetched) {
    int rc = fetch_locked(e, nullptr);
    if (rc) return rc;
  }
  const uint8_t reason = e->h_prefilter.as<uint8_t>()[pod];
  st->reason = reason;
  // batchscheduler.go:104-107: nil -> Success, any error -> Unschedulable
  st->code = reason == BS_PF_PASS ? BS_CODE_SUCCESS : BS_CODE_UNSCHEDULABLE;
  const int32_t g = e->h_gid[pod];
  st->group = (g >= 0 && (uint32_t)g < e->G) ? g : -1;
  return BS_OK;
}

int bs_permit(bs_engine* e, uint32_t pod, uint32_t node, bs_permit_result* r) {
  if (!e || !r) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->evaluated) return fail(e, BS_E_STATE, "bs_permit: evaluate first");
  if (pod >= e->P || node >= e->N) return BS_E_INDEX;
  if (!e->fetched) {
    int rc = fetch_locked(e, nullptr);
    if (rc) return rc;
  }
  const int64_t kSecond = 1000000000ll, kDefaultWait = 60 * kSecond;  // util.DefaultWaitTime k8s.go:31
  const int32_t g = e->h_gid[pod];
  memset(r, 0, sizeof(*r));
  r->group = -1;
  if (g == BS_GID_NONE) {  // core.go:270-272 + batchscheduler.go:190-193
    r->ready = 1;
    r->code = BS_CODE_SUCCESS;
    r->wait_ns = 0;
    return BS_OK;
  }
  if (g < 0 || (uint32_t)g >= e->G) {  // core.go:275-277 + batchscheduler.go:194-195
    r->ready = 0;
    r->code = BS_CODE_UNSCHEDULABLE;
    r->wait_ns = kDefaultWait;
    return BS_OK;
  }
  r->group = g;
  // util.GetWaitTimeDuration (k8s.go:82-91) + 1s (batchscheduler.go:180-182)
  int64_t wait = e->default_wait_ns;
  if ((size_t)g < e->h_wait_ns.size() && e->h_wait_ns[g] >= 0) wait = e->h_wait_ns[g];
  r->wait_ns = wait + kSecond;
  const uint8_t a = e->h_admit.as<uint8_t>()[g];
  r->ready = a == BS_ADMIT;              // core.go:303-307
  r->start_signal = r->ready;            // batchscheduler.go:197-199
  r->code = BS_CODE_WAIT;                // :184-187 and :201
  return BS_OK;
}

int bs_less(bs_engine* e, uint32_t a, uint32_t b) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->evaluated) return fail(e, BS_E_STATE, "bs_less: evaluate first");
  if (a >= e->P || b >= e->P) return BS_E_INDEX;
  if (!e->fetched) {
    int rc = fetch_locked(e, nullptr);
    if (rc) return rc;
  }
  // core.go:395-399: at equal priority, two grouped pods where a lister lookup fails
  // compare false both ways; everything else is the rank order of the device sort.
  auto miss = [&](uint32_t p) {
    const int32_t g = e->h_gid[p];
    return g != BS_GID_NONE && (g < 0 || (uint32_t)g >= e->G || (e->h_pflags[p] & BS_POD_LISTER_MISS));
  };
  if (e->h_prio[a] == e->h_prio[b] && e->h_gid[a] != BS_GID_NONE && e->h_gid[b] != BS_GID_NONE &&
      (miss(a) || miss(b)))
    return 0;
  const uint32_t* rank = e->h_rank.as<uint32_t>();
  return rank[a] < rank[b] ? 1 : 0;
}

int bs_format_message(const bs_status* st, const char* ns_name, const char* occupied_by, char* buf,
                      size_t buf_len) {
  if (!st || !buf || !buf_len) return BS_E_INVAL;
  const char* n = ns_name ? ns_name : "";
  const char* o = occupied_by ? occupied_by : "";
  switch (st->reason) {
    case BS_PF_PASS: snprintf(buf, buf_len, "%s", ""); break;
    case BS_PF_ERR_NOT_FOUND: snprintf(buf, buf_len, "can not found pod group: %s", n); break;           // core.go:102
    case BS_PF_ERR_DENIED: snprintf(buf, buf_len, "pod with pgName: %s last failed in 20s, deny", n); break;  // :107
    case BS_PF_ERR_OCCUPIED_NOREFS: snprintf(buf, buf_len, "pod group %s has been occupied by %s", n, o); break;  // :505
    case BS_PF_ERR_OCCUPIED: snprintf(buf, buf_len, "pod group has been occupied by %s", o); break;      // :509
    case BS_PF_ERR_NOT_ENOUGH: snprintf(buf, buf_len, "cluster resource not enough"); break;             // :143,:164
    default: return BS_E_INVAL;
  }
  return BS_OK;
}

// kube-scheduler v1.17.5's predicate reasons (restated) and FitError.Error(): "0/N nodes are available: " + the
// sorted "<count> <reason>" entries joined by ", " + "."
int bs_format_fit_error(const uint32_t* counts, uint32_t n_lanes, uint32_t n_nodes, const char* const* scalar_names,
                        char* buf, size_t buf_len) {
  return bs_format_fit_error_interpod(counts, n_lanes, nullptr, n_nodes, scalar_names, buf, buf_len);
}

int bs_format_fit_error_interpod(const uint32_t* counts, uint32_t n_lanes, const uint32_t* interpod, uint32_t n_nodes,
                                 const char* const* scalar_names, char* buf, size_t buf_len) {
  return bs_format_fit_error_filters(counts, n_lanes, interpod, nullptr, n_nodes, scalar_names, buf, buf_len);
}

int bs_format_fit_error_filters(const uint32_t* counts, uint32_t n_lanes, const uint32_t* interpod,
                                const uint32_t* host_ports, uint32_t n_nodes, const char* const* scalar_names, char* buf,
                                size_t buf_len) {
  if (!counts || !buf || !buf_len || n_lanes < BS_FIXED_LANES || n_lanes > BS_MAX_LANES) return BS_E_INVAL;
  static const char* const kFixed[4] = {"node(s) were unschedulable", "node(s) were unavailable",
                                        "node(s) didn't match node selector",
                                        "node(s) had taints that the pod didn't tolerate"};
  static const char* const kLane[4] = {"cpu", "memory", "ephemeral-storage", "pods"};
  std::vector<std::string> entries;
  for (uint32_t b = 0; b < 4 + n_lanes; ++b) {
    if (!counts[b]) continue;
    std::string text;
    if (b < 4) text = kFixed[b];
    else {
      const uint32_t d = b - 4;
      text = "Insufficient ";
      if (d < 4) text += kLane[d];
      else if (scalar_names && scalar_names[d - 4]) text += scalar_names[d - 4];
      else text += "lane" + std::to_string(d);
    }
    entries.push_back(std::to_string(counts[b]) + " " + text);
  }
  if (interpod) {   // a node failing MatchInterPodAffinity reports ErrPodAffinityNotMatch and the step's own reason
    static const char* const kIpf[3] = {"node(s) didn't satisfy existing pods anti-affinity rules",
                                        "node(s) didn't match pod affinity rules",
                                        "node(s) didn't match pod anti-affinity rules"};
    const uint64_t all = (uint64_t)interpod[0] + interpod[1] + interpod[2];
    if (all) entries.push_back(std::to_string(all) + " node(s) didn't match pod affinity/anti-affinity");
    for (int k = 0; k < 3; ++k)
      if (interpod[k]) entries.push_back(std::to_string(interpod[k]) + " " + kIpf[k]);
  }
  if (host_ports && host_ports[0])   // ErrPodNotFitsHostPorts
    entries.push_back(std::to_string(host_ports[0]) + " node(s) didn't have free ports for the requested pod ports");
  std::sort(entries.begin(), entries.end());   // byte-wise, as Go's sort.Strings
  std::string msg = "0/" + std::to_string(n_nodes) + " nodes are available: ";
  for (size_t k = 0; k < entries.size(); ++k) msg += (k ? ", " : "") + entries[k];
  msg += ".";
  if (msg.size() + 1 > buf_len) return BS_E_INVAL;
  memcpy(buf, msg.c_str(), msg.size() + 1);
  return BS_OK;
}

int bs_node_left(bs_engine* e, uint64_t sel, uint64_t tol, float percent, int64_t* left, uint32_t* present) {
  if (!e || !left || !present) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->have_nodes) return fail(e, BS_E_STATE, "bs_node_left: upload nodes first");
  BS_DEVICE_GUARD(e);
  const uint32_t N = e->N, L = e->L;
  if (!N) return BS_OK;
  DevBuf dl, dp;
  CK(dl.ensure((size_t)L * N * 8));
  CK(dp.ensure((size_t)N * 4));
  node_left_class_kernel<<<cdiv(N, 256), 256, 0, e->s>>>(node_tab(e), sel, tol, percent, dl.as<int64_t>(),
                                                         dp.as<uint32_t>());
  e->launches++;
  CK(cudaMemcpyAsync(left, dl.p, (size_t)L * N * 8, cudaMemcpyDeviceToHost, e->s));
  CK(cudaMemcpyAsync(present, dp.p, (size_t)N * 4, cudaMemcpyDeviceToHost, e->s));
  CK(cudaStreamSynchronize(e->s));
  return BS_OK;
}

int bs_cluster_check(bs_engine* e, uint64_t sel, uint64_t tol, float percent, const int64_t* need,
                     const uint32_t* need_present, uint32_t n_needs, uint8_t* ok) {
  if (!e || (n_needs && (!need || !need_present || !ok))) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->have_nodes) return fail(e, BS_E_STATE, "bs_cluster_check: upload nodes first");
  BS_DEVICE_GUARD(e);
  const uint32_t N = e->N, L = e->L;
  if (!n_needs) return BS_OK;
  if (!N) {
    memset(ok, 0, n_needs);  // empty snapshot list: the loop never runs (core.go:604,631)
    return BS_OK;
  }
  DevBuf scratch;
  View pre, pp, stats, dn, dnp, dok, spart, spres, scst, sdone;
  const size_t n_chunks = cdiv(N, PREFIX_CHUNK);
  CK(carve(scratch, {{&pre, (size_t)L * N * 8}, {&spart, n_chunks * BS_MAX_LANES * 8}, {&spres, n_chunks * 4},
                     {&scst, n_chunks * sizeof(ClassStats)}, {&sdone, 4}, {&pp, (size_t)N * 4}, {&stats, sizeof(ClassStats)},
                     {&dn, (size_t)L * n_needs * 8}, {&dnp, (size_t)n_needs * 4}, {&dok, n_needs}}));
  CK(cudaMemsetAsync(sdone.p, 0, 4, e->s));
  CK(cudaMemcpyAsync(dn.p, need, (size_t)L * n_needs * 8, cudaMemcpyHostToDevice, e->s));
  CK(cudaMemcpyAsync(dnp.p, need_present, (size_t)n_needs * 4, cudaMemcpyHostToDevice, e->s));
  PrefixOut po{pre.as<int64_t>(), pp.as<uint32_t>(), stats.as<ClassStats>()};
  NodeTab t = node_tab(e);
  PrefixSel ps{nullptr, nullptr, nullptr, 0, 2, sel, tol, percent, nullptr};
  PrefixScratch psc{spart.as<int64_t>(), spres.as<uint32_t>(), scst.as<ClassStats>(), sdone.as<uint32_t>()};
  launch_prefix(L, t, ps, psc, po, 1, e->s);
  const uint64_t threads = (uint64_t)n_needs * 32;
  needs_check_kernel<<<(uint32_t)((threads + 255) / 256), 256, 0, e->s>>>(
      t, po, dn.as<int64_t>(), dnp.as<uint32_t>(), n_needs, dok.as<uint8_t>());
  e->launches += 3;
  CK(cudaMemcpyAsync(ok, dok.p, n_needs, cudaMemcpyDeviceToHost, e->s));
  CK(cudaStreamSynchronize(e->s));
  CK(cudaGetLastError());
  return BS_OK;
}

namespace {
// bs_replay and bs_replay_priority (replay.cuh): the checks, the scratch copies, the walk and the read-back.  `scored`
// selects bs_replay_priority's node choice, which also needs both non-zero columns and reads the live node column back
// into nz_after ([2][N], or NULL).  The caller holds the engine's lock.
int replay_walk(bs_engine* e, const char* who, const uint32_t* queue, uint32_t n_queue, bs_replay_result* out,
                bool scored, int64_t* nz_after) {
  const std::string w(who);
  if (!e->have_nodes || !e->have_pods || !e->have_groups)
    return fail(e, BS_E_STATE, (w + ": upload nodes, groups and pods first").c_str());
  if (scored && !(e->nz.have_node && e->nz.have_pod))
    return fail(e, BS_E_STATE, (w + ": upload both non-zero request columns first").c_str());
  const bool loc = scored && (e->w_img || e->w_avoid);
  const bool hp = e->hp.on, ipf = e->ipf.on;
  int rc;
  if (loc && (rc = locality_check(e, who))) return rc;
  if (hp && (rc = host_port_check(e, who))) return rc;
  if (ipf && (rc = interpod_filter_check(e, who))) return rc;
  if (ipf && e->ipf.placed_term_max >= (int64_t)e->ipf.node.terms)
    return fail(e, BS_E_INDEX, (w + ": a placed class's term is outside the filter's term dictionary").c_str());
  BS_DEVICE_GUARD(e);
  const uint32_t N = e->N, Npad = e->Npad, P = e->P, G = e->G, L = e->L;
  if (!queue) n_queue = P;
  if (n_queue && (!out->prefilter || !out->node || !out->ready)) return BS_E_INVAL;
  if (queue)
    for (uint32_t i = 0; i < n_queue; ++i)
      if (queue[i] >= P) return fail(e, BS_E_INDEX, (w + ": queue entry is not a pod of the table").c_str());
  // the live non-zero sums: at most the node column's maximum plus every queued pod's
  for (int r = 0; r < 2 && scored; ++r)
    if ((long double)e->nz.node_max[r] + (long double)n_queue * (long double)e->nz.pod_max[r] > 0x1p62L)
      return fail(e, BS_E_RANGE, (w + ": live non-zero requests could pass 2^62").c_str());
  if (e->classes_dirty && (rc = rebuild_classes(e))) return rc;
  if (loc && (rc = locality_prepass(e))) return rc;
  if (ipf && e->ipf.dirty) {   // presence of the sides of now; the next evaluation builds its class fit bits again
    if ((rc = interpod_filter_prepass(e))) return rc;
    e->ipf.walk_prepass = true;
  }

  // scratch copies of everything the cycle mutates, the queue and the outputs, and the compact node state and
  // block cache the kernel builds (replay.cuh)
  const uint32_t Gp = std::max(G, 1u), Qp = std::max(n_queue, 1u);
  const bool fitmask = e->n_rep_classes <= (uint32_t)REPLAY_MAX_CLASSES;
  // block cache of the cluster scan: every running sum must stay below 2^62.  A pod is only assumed where it
  // fits, so a node's `requested` never passes its capacity by more than one request; only negative requests
  // accumulate without that limit.
  long double worst = 0;
  const NodeStats& ns = e->node_stats;
  const PodStats& ps = e->pod_stats;
  for (uint32_t d = 0; d < L; ++d)
    worst = std::max(worst, (long double)ns.max_alloc[d] + (long double)ns.max_requested[d] + (long double)ps.max_req[d] +
                                (long double)ps.neg_req[d] * (long double)n_queue + (long double)ns.max_pod_count + n_queue);
  const bool safe = worst * (long double)std::max(N, 1u) < 4.0e18L;
  const uint32_t n_blocks = cdiv(N, REPLAY_BLOCK);
  const bool cache = safe && fitmask && n_blocks >= 1 && n_blocks <= (uint32_t)REPLAY_MAX_BLOCKS;
  const size_t rows = cache ? (size_t)2 * e->n_rep_classes * n_blocks : 0;
  const size_t maxl = with_maxl<5, 9, 16>(L, [](auto M) { return (size_t)M; });   // launch_replay's lane bound
  View s_req, s_pc, s_rp, s_matched, s_gflags, s_grc, s_minres, s_mrp, d_queue, d_pf, d_node, d_ready, d_status,
      n_left0, n_left1, n_both, n_stat, n_fit, c_sum, c_max, c_keys, n_nz, s_used, d_want, d_conf, s_pres, s_hits,
      d_fclass;
  const InterpodNodeSide& is = e->ipf.node;
  const size_t ipf_words = ipf ? (is.slots + 31) / 32 : 0;
  // The node state and block cache every step reads come first: carved behind the copies, the same kernel took
  // 2 % longer at the bench shape on an H100.
  CK(carve(e->d_replay,
           {{&n_left0, (size_t)L * Npad * 8}, {&n_left1, (size_t)L * Npad * 8}, {&n_both, (size_t)Npad * 4},
            {&n_stat, Npad}, {&n_fit, fitmask ? (size_t)Npad * 4 : 0}, {&c_sum, rows * maxl * 8},
            {&c_max, rows * maxl * 8}, {&c_keys, rows * 4}, {&s_req, (size_t)L * Npad * 8}, {&s_pc, (size_t)Npad * 4},
            {&s_rp, (size_t)Npad * 4}, {&s_matched, (size_t)Gp * 4}, {&s_gflags, Gp}, {&s_grc, (size_t)Gp * 4},
            {&s_minres, (size_t)L * Gp * 8}, {&s_mrp, (size_t)Gp * 4}, {&d_queue, (size_t)Qp * 4}, {&d_pf, Qp},
            {&d_node, (size_t)Qp * 4}, {&d_ready, Qp}, {&d_status, 128}, {&n_nz, scored ? (size_t)2 * Npad * 8 : 0},
            {&s_used, hp ? (size_t)Npad * 8 : 0}, {&d_want, hp ? (size_t)P * 8 : 0}, {&d_conf, hp ? (size_t)P * 8 : 0},
            {&s_pres, ipf_words * 2 * 4}, {&s_hits, ipf ? (size_t)is.terms * 4 : 0},
            {&d_fclass, ipf ? (size_t)P * 4 : 0}}));
  auto dup = [&](const View& dst, const DevBuf& src, size_t bytes) {
    return bytes ? cudaMemcpyAsync(dst.p, src.p, bytes, cudaMemcpyDeviceToDevice, e->s) : cudaSuccess;
  };
  CK(dup(s_req, e->d_requested, (size_t)L * Npad * 8));
  CK(dup(s_pc, e->d_pod_count, (size_t)Npad * 4));
  CK(dup(s_rp, e->d_rpres, (size_t)Npad * 4));
  CK(dup(s_matched, e->d_matched, (size_t)G * 4));
  CK(dup(s_gflags, e->d_gflags, (size_t)G));
  CK(dup(s_grc, e->d_group_rep_class, (size_t)G * 4));
  CK(dup(s_minres, e->d_min_res, (size_t)L * G * 8));
  CK(dup(s_mrp, e->d_mrpres, (size_t)G * 4));
  if (scored) CK(dup(n_nz, e->nz.d_node, (size_t)2 * Npad * 8));
  std::vector<uint64_t> conf;   // each pod's conflict mask (host_port_check has passed: every want bit is an entry)
  if (hp) {
    CK(dup(s_used, e->hp.d_used, (size_t)Npad * 8));
    conf.assign(P, 0);
    for (uint32_t p = 0; p < P; ++p) conf[p] = hp_conflict_of(e, e->hp.h_want[p]);
    if (P) {
      CK(cudaMemcpyAsync(d_want.p, e->hp.h_want.data(), (size_t)P * 8, cudaMemcpyHostToDevice, e->s));
      CK(cudaMemcpyAsync(d_conf.p, conf.data(), (size_t)P * 8, cudaMemcpyHostToDevice, e->s));
    }
  }
  if (ipf) {   // the live presence starts as the snapshot's
    CK(dup(s_pres, e->ipf.d_presence, ipf_words * 2 * 4));
    CK(dup(s_hits, e->ipf.d_hits, (size_t)is.terms * 4));
    if (P) CK(cudaMemcpyAsync(d_fclass.p, e->ipf.h_class.data(), (size_t)P * 4, cudaMemcpyHostToDevice, e->s));
  }
  if (queue && n_queue) CK(cudaMemcpyAsync(d_queue.p, queue, (size_t)n_queue * 4, cudaMemcpyHostToDevice, e->s));
  CK(cudaMemsetAsync(d_status.p, 0, 128, e->s));
  ReplayIpfArgs la{};
  ReplayArgs& a = la;
  a.nt = node_tab(e);
  a.nt.requested = s_req.as<int64_t>();
  a.nt.pod_count = s_pc.as<int32_t>();
  a.nt.req_present = s_rp.as<uint32_t>();
  a.requested = s_req.as<int64_t>();
  a.pod_count = s_pc.as<int32_t>();
  a.req_present = s_rp.as<uint32_t>();
  a.pt = pod_tab(e);
  a.left[0] = n_left0.as<int64_t>();
  a.left[1] = n_left1.as<int64_t>();
  a.both = n_both.as<uint32_t>();
  a.nstat = n_stat.as<uint8_t>();
  a.fitmask = fitmask ? n_fit.as<uint32_t>() : nullptr;
  a.rsel = e->d_rsel.as<uint64_t>();
  a.rtol = e->d_rtol.as<uint64_t>();
  a.raff = e->d_raff.as<uint32_t>();
  a.n_rep = e->n_rep_classes;
  a.cache_ok = cache ? 1 : 0;
  if (cache) {
    a.blk_sum = c_sum.as<int64_t>();
    a.blk_max = c_max.as<int64_t>();
    a.blk_keys = c_keys.as<uint32_t>();
  }
  a.min_member = e->d_min_member.as<uint32_t>();
  a.scheduled = e->d_scheduled.as<uint32_t>();
  a.matched = s_matched.as<uint32_t>();
  a.gflags = s_gflags.as<uint8_t>();
  a.grc = s_grc.as<uint32_t>();
  a.min_res = s_minres.as<int64_t>();
  a.mrpres = s_mrp.as<uint32_t>();
  a.G = G;
  a.queue = queue ? d_queue.as<uint32_t>() : nullptr;
  a.n_queue = n_queue;
  a.prefilter = d_pf.as<uint8_t>();
  a.node = d_node.as<int32_t>();
  a.ready = d_ready.as<uint8_t>();
  a.status = d_status.as<int32_t>();
  if (scored) {
    a.nz_live = n_nz.as<int64_t>();
    a.pod_nz = e->nz.d_pod.as<int64_t>();
    a.w = e->weights;
    a.ratio = e->ratio;
  }
  if (loc) {
    la.il = e->loc.d_il.as<uint8_t>();
    la.avoid_mask = e->loc.d_avoid_mask.as<uint64_t>();
    la.loc_class = e->loc.d_class.as<uint32_t>();
    la.avoid_bit = e->loc.d_avoid_bit.as<uint8_t>();
    la.w_img = e->w_img;
    la.w_avoid = e->w_avoid;
  }
  if (hp) {
    la.hp_live = s_used.as<uint64_t>();
    la.hp_want = d_want.as<uint64_t>();
    la.hp_conf = d_conf.as<uint64_t>();
  }
  if (ipf) {
    la.ipf_mbits = s_pres.as<uint32_t>();
    la.ipf_obits = s_pres.as<uint32_t>() + ipf_words;
    la.ipf_hits = s_hits.as<uint32_t>();
    la.tp = IpfTopo{is.d_topo.as<uint32_t>(), is.d_term_key.as<uint32_t>(), is.d_term_off.as<uint32_t>(), N};
    la.fc = IpfPods{e->ipf.d_poff.as<uint32_t>(), e->ipf.d_pterm.as<uint32_t>(), e->ipf.d_prole.as<uint8_t>(),
                    e->ipf.d_pself.as<uint8_t>(), e->ipf.pclasses};
    la.f_class = d_fclass.as<uint32_t>();
    la.q_class = e->ipf.d_qclass.as<uint32_t>();
    la.q_off = e->ipf.d_qoff.as<uint32_t>();
    la.q_term = e->ipf.d_qterm.as<uint32_t>();
    la.q_own = e->ipf.d_qown.as<int32_t>();
    la.q_match = e->ipf.d_qmatch.as<uint8_t>();
  }
  {
    StageTimer tm(e, BS_K_REPLAY, e->s);
    const uint32_t build = (scored ? REPLAY_SCORED : 0u) | (scored && e->ratio.weight ? REPLAY_RATIO : 0u) |
                           (loc ? REPLAY_LOC : 0u) | (hp ? REPLAY_HP : 0u) | (ipf ? REPLAY_IPF : 0u);
    launch_replay(L, build, la, e->s);
    tm.launched();
    CK(cudaGetLastError());
  }
  int32_t status[3] = {};   // panic, final lo, monotone
  std::vector<uint32_t> grc;
  auto d2h = [&](void* dst, const View& src, size_t bytes) {
    return dst && bytes ? cudaMemcpyAsync(dst, src.p, bytes, cudaMemcpyDeviceToHost, e->s) : cudaSuccess;
  };
  CK(d2h(status, d_status, sizeof(status)));
  CK(d2h(out->prefilter, d_pf, n_queue));
  CK(d2h(out->node, d_node, (size_t)n_queue * 4));
  CK(d2h(out->ready, d_ready, n_queue));
  if (out->node_requested && N)
    CK(cudaMemcpy2DAsync(out->node_requested, (size_t)N * 8, s_req.p, (size_t)Npad * 8, (size_t)N * 8, L,
                         cudaMemcpyDeviceToHost, e->s));
  CK(d2h(out->node_pod_count, s_pc, (size_t)N * 4));
  CK(d2h(out->node_req_present, s_rp, (size_t)N * 4));
  CK(d2h(out->group_matched, s_matched, (size_t)G * 4));
  CK(d2h(out->group_flags, s_gflags, (size_t)G));
  CK(d2h(out->group_min_res, s_minres, (size_t)L * G * 8));
  CK(d2h(out->group_min_res_present, s_mrp, (size_t)G * 4));
  if (scored && nz_after && N)
    CK(cudaMemcpy2DAsync(nz_after, (size_t)N * 8, n_nz.p, (size_t)Npad * 8, (size_t)N * 8, 2, cudaMemcpyDeviceToHost,
                         e->s));
  if (out->group_rep_sel || out->group_rep_tol) {
    grc.resize(Gp);
    CK(d2h(grc.data(), s_grc, (size_t)G * 4));
  }
  CK(cudaStreamSynchronize(e->s));
  {
    // the findMaxPG buckets as replay_kernel cuts them
    const uint32_t per = cdiv(G, 32u * REPLAY_MAX_BUCKETS), S = 32u * std::max(per, 1u);
    e->replay_shape = {true, cache, fitmask, e->n_rep_classes, n_blocks, S, cdiv(G, S), (uint32_t)status[1],
                       (uint32_t)status[2]};
  }
  if (status[0]) return fail(e, BS_E_REF_PANIC, (w + ": findMaxPG would divide by MinMember == 0 (core.go:716)").c_str());
  for (uint32_t g = 0; g < G && (out->group_rep_sel || out->group_rep_tol); ++g) {
    const ClassKey& k = e->rep_index.keys[grc[g]];
    if (out->group_rep_sel) out->group_rep_sel[g] = k.sel;
    if (out->group_rep_tol) out->group_rep_tol[g] = k.tol;
  }
  return BS_OK;
}
}  // namespace

// The walks follow their own placements in live MatchInterPodAffinity presence, which needs each pod's placed class:
// without it they refuse.
static int interpod_placed_refuse(bs_engine* e, const char* who) {
  return fail(e, BS_E_INVAL, (std::string(who) + ": the MatchInterPodAffinity filter needs the pods' placed classes in "
                              "the walk; upload them with bs_upload_pod_interpod_placed or switch the filter off with "
                              "bs_set_interpod_filter").c_str());
}

int bs_replay(bs_engine* e, const uint32_t* queue, uint32_t n_queue, bs_replay_result* out) {
  if (!e || !out) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  if (e->ipf.on && !e->ipf.have_placed) return interpod_placed_refuse(e, "bs_replay");
  return replay_walk(e, "bs_replay", queue, n_queue, out, false, nullptr);
}

int bs_replay_priority(bs_engine* e, const uint32_t* queue, uint32_t n_queue, bs_replay_result* out,
                       int64_t* node_nonzero_after) {
  if (!e || !out) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  if (e->ipf.on && !e->ipf.have_placed) return interpod_placed_refuse(e, "bs_replay_priority");
  if (e->w_taint || e->w_naff)   // their maxima would have to follow the walk's live fit set, which is not built yet
    return fail(e, BS_E_INVAL, "bs_replay_priority: TaintToleration and NodeAffinity are not supported in the walk; "
                               "set both weights of bs_set_node_priority_weights to 0");
  if (e->w_spread)   // its maxima and zone sums would follow the live fit set and the live counts, likewise
    return fail(e, BS_E_INVAL, "bs_replay_priority: SelectorSpread is not supported in the walk; "
                               "set bs_set_spread_weight to 0");
  if (e->w_ipa)   // its maxima would follow the live fit set and the live placements, likewise
    return fail(e, BS_E_INVAL, "bs_replay_priority: InterPodAffinity is not supported in the walk; "
                               "set bs_set_interpod_weight to 0");
  return replay_walk(e, "bs_replay_priority", queue, n_queue, out, true, node_nonzero_after);
}

// ---- preemption: bs_upload_bound_pods, bs_preempt, bs_remove_pod (preempt.cuh) ----
int bs_upload_bound_pods(bs_engine* e, const bs_bound_table* t) {
  if (!e || !t) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->have_nodes) return fail(e, BS_E_STATE, "bs_upload_bound_pods: upload nodes first");
  if (t->n_lanes != e->L) return fail(e, BS_E_INVAL, "bs_upload_bound_pods: n_lanes differs from the engine's");
  const uint32_t V = t->n_pods, L = e->L, N = e->N;
  if (V && (!t->node || !t->req || !t->req_present || !t->gid || !t->priority || !t->start_ns || !t->flags))
    return fail(e, BS_E_INVAL, "bs_upload_bound_pods: null column");
  e->have_bound = e->hp.have_bound = false;   // a failing table is dropped, and the host-port masks go with it
  // rows: node index, scalar keys within the node's, value range
  BoundStats bs = Chunks(V, 8192).reduce<BoundStats>([&](int, uint32_t a0, uint32_t a1, BoundStats& st) {
    for (uint32_t v = a0; v < a1; ++v) {
      const uint32_t n = t->node[v];
      if (n >= N) { st.bad_index = true; continue; }
      st.bad_keys = st.bad_keys || (t->req_present[v] & ~0xFu & ~e->h_nrpres[n]) != 0;
      st.max_gid = std::max(st.max_gid, t->gid[v]);
      st.bad_index = st.bad_index || t->gid[v] < BS_GID_MISSING;   // neither a group, BS_GID_NONE nor BS_GID_MISSING
    }
    for (uint32_t d = 0; d < L; ++d) {
      if (d == (uint32_t)LANE_PODS) continue;
      const int64_t* r = t->req + (size_t)d * V;
      int64_t lo = 0, hi = 0;
      for (uint32_t v = a0; v < a1; ++v) { lo = std::min(lo, r[v]); hi = std::max(hi, r[v]); }
      st.bad_range = st.bad_range || lo < -BS_VALUE_LIMIT || hi > BS_VALUE_LIMIT;
    }
  });
  if (bs.bad_index) return fail(e, BS_E_INDEX, "bs_upload_bound_pods: node index outside the snapshot or gid < BS_GID_MISSING");
  // CSR by node
  std::vector<uint32_t> row(N + 1, 0), order(V);
  for (uint32_t v = 0; v < V; ++v) row[t->node[v] + 1]++;
  for (uint32_t n = 0; n < N; ++n) {
    bs.bad_count = bs.bad_count || (int64_t)row[n + 1] > (int64_t)e->h_npc[n];
    row[n + 1] += row[n];
  }
  if (bs.bad_count) return fail(e, BS_E_INVAL, "bs_upload_bound_pods: more bound pods on a node than its pod_count");
  if (bs.bad_keys) return fail(e, BS_E_INVAL, "bs_upload_bound_pods: scalar keys outside the node's req_present");
  if (bs.bad_range) return fail(e, BS_E_RANGE, "bs_upload_bound_pods: value outside +-2^56");
  {
    std::vector<uint32_t> fill(row.begin(), row.end() - 1);
    for (uint32_t v = 0; v < V; ++v) order[fill[t->node[v]]++] = v;   // table order within a node
  }
  // per node: MoreImportantPod order (priority descending, start ascending, index ascending) and the suffix range
  const int64_t* req = t->req;
  const bool suffix_bad = Chunks(N, 1024).reduce<BoundStats>([&](int, uint32_t n0, uint32_t n1, BoundStats& st) {
    for (uint32_t n = n0; n < n1; ++n) {
      uint32_t* a = order.data() + row[n];
      std::sort(a, order.data() + row[n + 1], [&](uint32_t x, uint32_t y) {
        if (t->priority[x] != t->priority[y]) return t->priority[x] > t->priority[y];
        if (t->start_ns[x] != t->start_ns[y]) return t->start_ns[x] < t->start_ns[y];
        return x < y;
      });
      for (uint32_t d = 0; d < L && !st.bad_range; ++d) {
        if (d == (uint32_t)LANE_PODS) continue;
        int64_t s = 0;
        for (uint32_t k = row[n + 1]; k-- > row[n];) {
          const uint32_t v = order[k];
          if (d >= 4 && !((t->req_present[v] >> d) & 1u)) continue;
          s += req[(size_t)d * V + v];
          st.bad_range = st.bad_range || s < -BS_VALUE_LIMIT || s > BS_VALUE_LIMIT;
        }
      }
    }
  }).bad_range;
  if (suffix_bad) return fail(e, BS_E_RANGE, "bs_upload_bound_pods: a per-node suffix sum outside +-2^56");
  // columns in CSR order: lane 3 and scalar lanes the row has no key for are not removed
  const size_t Vp = std::max(V, 1u);
  std::vector<int32_t> prio(Vp, 0), gid(Vp, 0);
  std::vector<int64_t> start(Vp, 0), breq((size_t)L * Vp, 0);
  std::vector<uint8_t> flags(Vp, 0);
  Chunks(V, 8192).run([&](int, uint32_t k0, uint32_t k1) {
    for (uint32_t k = k0; k < k1; ++k) {
      const uint32_t v = order[k];
      prio[k] = t->priority[v];
      gid[k] = t->gid[v];
      start[k] = t->start_ns[v];
      flags[k] = t->flags[v];
      for (uint32_t d = 0; d < L; ++d)
        if (d != (uint32_t)LANE_PODS && (d < 4 || ((t->req_present[v] >> d) & 1u))) breq[(size_t)d * V + k] = req[(size_t)d * V + v];
    }
  });
  BS_DEVICE_GUARD(e);
  int rc;
  if ((rc = upload_vec(e, e->d_brow, row.data(), N + 1, N + 1))) return rc;
  if ((rc = upload_vec(e, e->d_bprio, prio.data(), V, (uint32_t)Vp))) return rc;
  if ((rc = upload_vec(e, e->d_bstart, start.data(), V, (uint32_t)Vp))) return rc;
  if ((rc = upload_vec(e, e->d_bgid, gid.data(), V, (uint32_t)Vp))) return rc;
  if ((rc = upload_vec(e, e->d_bflags, flags.data(), V, (uint32_t)Vp))) return rc;
  if ((rc = upload_vec(e, e->d_bidx, order.data(), V, (uint32_t)Vp))) return rc;
  if ((rc = upload_col(e, col(breq.data(), e->d_breq, L), (uint32_t)Vp, (uint32_t)Vp))) return rc;
  CK(e->d_bsuf.ensure((size_t)L * Vp * 8));
  CK(e->d_bsuf_online.ensure(Vp * 4));
  CK(e->d_bsuf_bad.ensure(Vp * 4));
  CK(e->d_bsuf_vio.ensure(Vp * 4));
  // the residuals the bound table is read against: node_left_kernel with no lane-class tables, into buffers of
  // its own (the round's tables stay as they are)
  CK(e->d_pl_left.ensure((size_t)L * e->Npad * 8));
  CK(e->d_pl_present.ensure((size_t)e->Npad * 4));
  if (N) {
    preempt_prep_kernel<<<cdiv(N, 256), 256, 0, e->s>>>(e->d_brow.as<uint32_t>(), e->d_bgid.as<int32_t>(),
                                                       e->d_bflags.as<uint8_t>(), e->d_breq.as<int64_t>(),
                                                       e->d_bsuf.as<int64_t>(), e->d_bsuf_online.as<uint32_t>(),
                                                       e->d_bsuf_bad.as<uint32_t>(), e->d_bsuf_vio.as<uint32_t>(), N,
                                                       (uint32_t)Vp, L);
    ++e->launches;
  }
  node_left_kernel<<<cdiv(e->Npad, 256), 256, 0, e->s>>>(node_tab(e), LaneMap{}, nullptr, nullptr,
                                                         e->d_pl_present.as<uint32_t>(), nullptr,
                                                         e->d_pl_left.as<int64_t>());
  ++e->launches;
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(e->s));   // the host vectors die here
  e->h_bgid.assign(t->gid, t->gid + V);
  e->h_bnode.assign(t->node, t->node + V);
  e->h_bflags.assign(t->flags, t->flags + V);
  e->V = V;
  e->bound_max_gid = bs.max_gid;
  e->have_bound = true;
  return BS_OK;
}

namespace {
// What bs_preempt and bs_preempt_walk hand their kernels for each preemptor: its row, and while the PodFitsHostPorts
// filter is on (hp) its conflict mask and, in the walk, its want mask (what its nomination adds to its node's).
struct Preemptors {
  bool hp = false;
  std::vector<PreemptPod> pp;
  std::vector<uint64_t> conf, want;
};

// bs_preempt's and bs_preempt_walk's checks, in this order: the arguments; the MatchInterPodAffinity filter, which
// preemption refuses (its presence would have to shrink when victims leave: upstream's metadata RemovePod); the
// PodFitsHostPorts filter without the bound pods' host-port masks (bs_upload_bound_host_ports), which preemption needs
// to take its victims' ports out of the used masks; flag bits other than BS_PREEMPT_GANG; both sides of the ports
// filter as the round needs them, and each bound row's bits entries of the node side's dictionary that its node uses
// (a NodeInfo's used ports include its pods'); the tables; each preemptor.  `walk` fills q.want.  The caller holds the
// engine's lock.
int preempt_prologue(bs_engine* e, const char* who, const uint32_t* pods, uint32_t n, const bs_preempt_result* out,
                     uint32_t flags, bool walk, Preemptors& q) {
  if (!out || (n && (!pods || !out->node || !out->n_victims || !out->n_candidates)) || !out->victim_offset)
    return BS_E_INVAL;
  const Refuse bad{e, who};
  if (e->ipf.on)
    return bad(BS_E_INVAL, "the MatchInterPodAffinity filter is not supported here; switch it off with "
                           "bs_set_interpod_filter");
  q.hp = e->hp.on;
  if (q.hp && !e->hp.have_bound)
    return bad(BS_E_INVAL, "the PodFitsHostPorts filter needs the bound pods' host ports in preemption; upload them "
                           "with bs_upload_bound_host_ports or switch the filter off with bs_set_host_port_filter");
  if (flags & ~BS_PREEMPT_GANG) return bad(BS_E_INVAL, "unknown flag bits");
  if (q.hp) {
    if (int rc = host_port_check(e, who)) return rc;
    const std::vector<uint64_t>& bp = e->hp.h_bports;
    uint64_t all = 0;
    bool outside = false;
    for (uint32_t v = 0; v < (uint32_t)bp.size(); ++v) {
      all |= bp[v];
      outside = outside || (bp[v] & ~e->hp.h_used[e->h_bnode[v]]) != 0;
    }
    if (e->hp.entries < 64 && (all >> e->hp.entries))
      return bad(BS_E_INDEX, "a bound pod's host-port bit is outside the node side's dictionary");
    if (outside) return bad(BS_E_INVAL, "a bound pod holds a host port its node's used mask does not have");
  }
  if (!e->have_nodes || !e->have_groups || !e->have_pods || !e->have_bound)
    return bad(BS_E_STATE, "upload nodes, groups, pods and the bound-pod table first");
  if (e->bound_max_gid >= (int32_t)e->G) return bad(BS_E_INDEX, "a bound pod's group index >= n_groups");
  q.pp.assign(std::max(n, 1u), PreemptPod{});
  if (q.hp) q.conf.assign(std::max(n, 1u), 0);
  if (q.hp && walk) q.want.assign(std::max(n, 1u), 0);
  for (uint32_t i = 0; i < n; ++i) {
    const uint32_t p = pods[i];
    if (p >= e->P) return bad(BS_E_INDEX, "pod index outside the pod table");
    const ClassKey& k = e->fit_index.keys[e->h_pfc[p]];
    if (k.aff != BS_AFF_NONE && k.aff >= e->n_aff) return bad(BS_E_INDEX, "affinity class outside the uploaded table");
    q.pp[i] = PreemptPod{k.sel, k.tol, p, k.nz, k.aff, e->h_prio[p], e->h_gid[p]};
    if (q.hp) q.conf[i] = hp_conflict_of(e, e->hp.h_want[p]);
    if (q.hp && walk) q.want[i] = e->hp.h_want[p];
  }
  return BS_OK;
}

// The kernels' view of the uploaded node and bound tables and of the preemptors in e->d_pp.
PreemptArgs preempt_args(const bs_engine* e, uint32_t n) {
  PreemptArgs a{};
  a.t = node_tab(e);
  a.left = e->d_pl_left.as<int64_t>();
  a.left_present = e->d_pl_present.as<uint32_t>();
  a.b = BoundTab{e->d_brow.as<uint32_t>(), e->d_brow.as<uint32_t>() + 1, e->d_bprio.as<int32_t>(),
                 e->d_bstart.as<int64_t>(), e->d_bgid.as<int32_t>(), e->d_bflags.as<uint8_t>(), e->d_bidx.as<uint32_t>(),
                 e->d_breq.as<int64_t>(), e->d_bsuf.as<int64_t>(), e->d_bsuf_online.as<uint32_t>(),
                 e->d_bsuf_bad.as<uint32_t>(), e->d_bsuf_vio.as<uint32_t>(), std::max(e->V, 1u)};
  a.pp = e->d_pp.as<PreemptPod>();
  a.preq = e->d_req.as<int64_t>();
  a.preq_present = e->d_ppres.as<uint32_t>();
  a.P = e->P;
  a.n = n;
  a.n_tiles = cdiv(e->N, PREEMPT_THREADS);
  return a;
}

// The PodFitsHostPorts views of PreemptHpArgs: bs_preempt passes the uploaded masks and no nominated or want masks,
// bs_preempt_walk its live copies.
void hp_views(PreemptHpArgs& ha, const uint64_t* used, const uint64_t* nom, const uint64_t* ports, const uint64_t* suf,
              const uint64_t* conf, const uint64_t* want) {
  ha.hp_used = used;
  ha.hp_nom = nom;
  ha.hp_ports = ports;
  ha.hp_suf = suf;
  ha.hp_conf = conf;
  ha.hp_want = want;
}
}  // namespace

int bs_preempt(bs_engine* e, const uint32_t* pods, uint32_t n, bs_preempt_result* out) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  Preemptors q;
  if (int rc = preempt_prologue(e, "bs_preempt", pods, n, out, 0, false, q)) return rc;
  const uint32_t L = e->L, N = e->N;
  out->victim_offset[0] = 0;
  out->victims_total = 0;
  if (!n) return BS_OK;
  BS_DEVICE_GUARD(e);
  CK(e->d_pp.ensure((size_t)n * sizeof(PreemptPod)));
  CK(e->d_pnode.ensure((size_t)n * 4));
  CK(e->d_pnv.ensure((size_t)n * 4));
  CK(e->d_pcand.ensure((size_t)n * 4));
  CK(e->d_poff.ensure((size_t)n * 4));
  CK(cudaMemcpyAsync(e->d_pp.p, q.pp.data(), (size_t)n * sizeof(PreemptPod), cudaMemcpyHostToDevice, e->s));
  PreemptHpArgs ha{};
  PreemptArgs& a = ha;
  a = preempt_args(e, n);
  if (q.hp) {
    CK(e->hp.d_pconf.ensure((size_t)n * 8));
    CK(cudaMemcpyAsync(e->hp.d_pconf.p, q.conf.data(), (size_t)n * 8, cudaMemcpyHostToDevice, e->s));
    hp_views(ha, e->hp.d_used.as<uint64_t>(), nullptr, e->hp.d_bports.as<uint64_t>(), e->hp.d_bsuf.as<uint64_t>(),
             e->hp.d_pconf.as<uint64_t>(), nullptr);
  }
  a.out_node = e->d_pnode.as<int32_t>();
  a.out_nv = e->d_pnv.as<uint32_t>();
  a.out_cand = e->d_pcand.as<uint32_t>();
  if (!N) {
    CK(cudaMemsetAsync(a.out_node, 0xff, (size_t)n * 4, e->s));
    CK(cudaMemsetAsync(a.out_nv, 0, (size_t)n * 4, e->s));
    CK(cudaMemsetAsync(a.out_cand, 0, (size_t)n * 4, e->s));
  } else {
    // preemptors in chunks: one grid row each (gridDim.y <= 65535), per-tile keys within a 256 MiB budget
    const size_t per = (size_t)a.n_tiles * sizeof(PickKey);
    const uint32_t chunk = (uint32_t)std::max<size_t>(1, std::min<size_t>({(size_t)65535, (size_t)n, ((size_t)256 << 20) / per}));
    CK(e->d_ptiles.ensure((size_t)chunk * per));
    a.tiles = e->d_ptiles.as<PickKey>();
    for (uint32_t p0 = 0; p0 < n; p0 += chunk) {
      const uint32_t cnt = std::min(chunk, n - p0);
      a.p0 = p0;
      with_preempt_build(L, q.hp, [&](auto M, auto H) {
        preempt_node_kernel<M, H><<<dim3(a.n_tiles, cnt), PREEMPT_THREADS, 0, e->s>>>(PreemptArgsOf<H>(ha));
      });
      preempt_reduce_kernel<<<cdiv(cnt, 256), 256, 0, e->s>>>(a, cnt);
      e->launches += 2;
    }
  }
  return preempt_read_back(e, "bs_preempt", a, n, out, [] { return BS_OK; }, [&](uint64_t total) -> int {
    CK(e->d_pvict.ensure((size_t)total * 4));
    CK(cudaMemcpyAsync(e->d_poff.p, out->victim_offset, (size_t)n * 4, cudaMemcpyHostToDevice, e->s));
    a.offset = e->d_poff.as<uint32_t>();
    a.victims = e->d_pvict.as<uint32_t>();
    with_preempt_build(L, q.hp, [&](auto M, auto H) {
      preempt_emit_kernel<M, H><<<dim3(cdiv(n, 256)), 256, 0, e->s>>>(PreemptArgsOf<H>(ha));
    });
    ++e->launches;
    CK(cudaGetLastError());
    return BS_OK;
  });
}

int bs_preempt_walk(bs_engine* e, const uint32_t* pods, uint32_t n, uint32_t flags, bs_preempt_result* out,
                    uint32_t* outcome, int32_t* evicted_by) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  Preemptors q;
  if (int rc = preempt_prologue(e, "bs_preempt_walk", pods, n, out, flags, true, q)) return rc;
  const bool gang = flags & BS_PREEMPT_GANG, hp = q.hp;
  const std::vector<PreemptPod>& pp = q.pp;
  // queue order: every earlier nomination has a priority >= the current preemptor's, so all of them count
  // (addNominatedPods) and none is ever cleared (getLowerPriorityNominatedPods)
  std::vector<uint8_t> seen(e->P, 0), closed(gang ? e->G : 0, 0), unit_last(std::max(n, 1u), 1);
  for (uint32_t i = 0; i < n; ++i) {
    if (i && pp[i].prio > pp[i - 1].prio)
      return fail(e, BS_E_INVAL, "bs_preempt_walk: priorities must be non-increasing along the list");
    if (seen[pp[i].pod]++) return fail(e, BS_E_INVAL, "bs_preempt_walk: a pod is listed twice");
    // a group index >= n_groups names no group of the table: like BS_GID_MISSING, a unit of one
    if (!gang || pp[i].gid < 0 || pp[i].gid >= (int32_t)e->G) continue;
    const int32_t g = pp[i].gid;
    if (i && pp[i - 1].gid == g) {
      unit_last[i - 1] = 0;
    } else {
      if (closed[g]) return fail(e, BS_E_INVAL, "bs_preempt_walk: the preemptors of a group are not contiguous");
      closed[g] = 1;
    }
  }
  // the live sums: nominations add requests (negative ones without the fit's bound) and pods
  const NodeStats& ns = e->node_stats;
  const PodStats& ps = e->pod_stats;
  for (uint32_t d = 0; d < e->L; ++d)
    if ((long double)ns.max_alloc[d] + (long double)ns.max_requested[d] + (long double)ps.max_req[d] +
            (long double)ps.neg_req[d] * (long double)n + (long double)ns.max_pod_count + n + (long double)BS_VALUE_LIMIT >
        0x1p62L)
      return fail(e, BS_E_RANGE, "bs_preempt_walk: live requests could pass 2^62");
  const uint32_t L = e->L, N = e->N, Npad = e->Npad, V = e->V, Vp = std::max(V, 1u);
  if (evicted_by) std::fill(evicted_by, evicted_by + V, -1);
  out->victim_offset[0] = 0;
  out->victims_total = 0;
  if (!n) return BS_OK;
  BS_DEVICE_GUARD(e);
  PreemptHpArgs ha{};
  PreemptArgs& a = ha;
  a = preempt_args(e, n);
  const size_t g_n = gang ? n : 0, g_v = gang ? Vp : 0, h_n = hp ? n : 0, h_v = hp ? Vp : 0;
  View w_pp, w_node, w_nv, w_cand, w_outcome, w_last, w_tiles, w_vict, w_ctl, w_end, w_prio, w_start, w_gid, w_flags,
      w_idx, w_req, w_suf, w_son, w_sbad, w_svio, w_requested, w_rp, w_pc, w_left, w_lp, w_evby, e_node, e_end, e_nv,
      e_row, e_req, e_rp, e_pc, r_pos, r_prio, r_start, r_gid, r_flags, r_idx, r_req, h_conf, h_want, h_used, h_nom,
      h_ports, h_suf, he_used, he_nom, hr_ports;
  CK(carve(e->d_walk,
           {{&w_pp, (size_t)n * sizeof(PreemptPod)}, {&w_node, (size_t)n * 4}, {&w_nv, (size_t)n * 4},
            {&w_cand, (size_t)n * 4}, {&w_outcome, (size_t)n * 4}, {&w_last, n}, {&w_tiles, a.n_tiles * sizeof(PickKey)},
            {&w_vict, (size_t)Vp * 4}, {&w_ctl, sizeof(WalkCtl)}, {&w_end, (size_t)N * 4}, {&w_prio, (size_t)Vp * 4},
            {&w_start, (size_t)Vp * 8}, {&w_gid, (size_t)Vp * 4}, {&w_flags, Vp}, {&w_idx, (size_t)Vp * 4},
            {&w_req, (size_t)L * Vp * 8}, {&w_suf, (size_t)L * Vp * 8}, {&w_son, (size_t)Vp * 4},
            {&w_sbad, (size_t)Vp * 4}, {&w_svio, (size_t)Vp * 4}, {&w_requested, (size_t)L * Npad * 8},
            {&w_rp, (size_t)Npad * 4}, {&w_pc, (size_t)Npad * 4}, {&w_left, (size_t)L * Npad * 8},
            {&w_lp, (size_t)Npad * 4}, {&w_evby, (size_t)Vp * 4}, {&e_node, g_n * 4}, {&e_end, g_n * 4},
            {&e_nv, g_n * 4}, {&e_row, g_n * 4}, {&e_req, L * g_n * 8}, {&e_rp, g_n * 4}, {&e_pc, g_n * 4},
            {&r_pos, g_v * 4}, {&r_prio, g_v * 4}, {&r_start, g_v * 8}, {&r_gid, g_v * 4}, {&r_flags, g_v},
            {&r_idx, g_v * 4}, {&r_req, L * g_v * 8}, {&h_conf, h_n * 8}, {&h_want, h_n * 8},
            {&h_used, hp ? (size_t)Npad * 8 : 0}, {&h_nom, hp ? (size_t)Npad * 8 : 0}, {&h_ports, h_v * 8},
            {&h_suf, h_v * 8}, {&he_used, hp ? g_n * 8 : 0}, {&he_nom, hp ? g_n * 8 : 0},
            {&hr_ports, hp ? g_v * 8 : 0}}));
  auto dup = [&](const View& dst, const void* src, size_t bytes) {
    return bytes ? cudaMemcpyAsync(dst.p, src, bytes, cudaMemcpyDeviceToDevice, e->s) : cudaSuccess;
  };
  CK(cudaMemcpyAsync(w_pp.p, pp.data(), (size_t)n * sizeof(PreemptPod), cudaMemcpyHostToDevice, e->s));
  CK(cudaMemcpyAsync(w_last.p, unit_last.data(), n, cudaMemcpyHostToDevice, e->s));
  CK(cudaMemsetAsync(w_ctl.p, 0, sizeof(WalkCtl), e->s));
  CK(cudaMemsetAsync(w_evby.p, 0xff, (size_t)Vp * 4, e->s));
  CK(dup(w_end, e->d_brow.as<uint32_t>() + 1, (size_t)N * 4));
  CK(dup(w_prio, e->d_bprio.p, (size_t)Vp * 4));
  CK(dup(w_start, e->d_bstart.p, (size_t)Vp * 8));
  CK(dup(w_gid, e->d_bgid.p, (size_t)Vp * 4));
  CK(dup(w_flags, e->d_bflags.p, Vp));
  CK(dup(w_idx, e->d_bidx.p, (size_t)Vp * 4));
  CK(dup(w_req, e->d_breq.p, (size_t)L * Vp * 8));
  CK(dup(w_suf, e->d_bsuf.p, (size_t)L * Vp * 8));
  CK(dup(w_son, e->d_bsuf_online.p, (size_t)Vp * 4));
  CK(dup(w_sbad, e->d_bsuf_bad.p, (size_t)Vp * 4));
  CK(dup(w_svio, e->d_bsuf_vio.p, (size_t)Vp * 4));
  CK(dup(w_requested, e->d_requested.p, (size_t)L * Npad * 8));
  CK(dup(w_rp, e->d_rpres.p, (size_t)Npad * 4));
  CK(dup(w_pc, e->d_pod_count.p, (size_t)Npad * 4));
  CK(dup(w_left, e->d_pl_left.p, (size_t)L * Npad * 8));
  CK(dup(w_lp, e->d_pl_present.p, (size_t)Npad * 4));
  WalkHpArgs hw{};
  WalkArgs& w = hw;
  w.end = w_end.as<uint32_t>();
  w.prio = w_prio.as<int32_t>();
  w.start = w_start.as<int64_t>();
  w.gid = w_gid.as<int32_t>();
  w.flags = w_flags.as<uint8_t>();
  w.idx = w_idx.as<uint32_t>();
  w.req = w_req.as<int64_t>();
  w.suf = w_suf.as<int64_t>();
  w.suf_online = w_son.as<uint32_t>();
  w.suf_bad = w_sbad.as<uint32_t>();
  w.suf_vio = w_svio.as<uint32_t>();
  w.requested = w_requested.as<int64_t>();
  w.req_present = w_rp.as<uint32_t>();
  w.pod_count = w_pc.as<int32_t>();
  w.left = w_left.as<int64_t>();
  w.left_present = w_lp.as<uint32_t>();
  w.evicted_by = w_evby.as<int32_t>();
  w.outcome = w_outcome.as<uint32_t>();
  w.unit_last = w_last.as<uint8_t>();
  w.ctl = w_ctl.as<WalkCtl>();
  if (gang) {
    w.ent_node = e_node.as<uint32_t>();
    w.ent_end = e_end.as<uint32_t>();
    w.ent_nv = e_nv.as<uint32_t>();
    w.ent_row = e_row.as<uint32_t>();
    w.ent_req = e_req.as<int64_t>();
    w.ent_rp = e_rp.as<uint32_t>();
    w.ent_pc = e_pc.as<int32_t>();
    w.row_pos = r_pos.as<uint32_t>();
    w.row_prio = r_prio.as<int32_t>();
    w.row_start = r_start.as<int64_t>();
    w.row_gid = r_gid.as<int32_t>();
    w.row_flags = r_flags.as<uint8_t>();
    w.row_idx = r_idx.as<uint32_t>();
    w.row_req = r_req.as<int64_t>();
  }
  w.n = n;
  // the kernels read the live state through PreemptArgs' views
  a.t.requested = w.requested;
  a.t.req_present = w.req_present;
  a.t.pod_count = w.pod_count;
  a.left = w.left;
  a.left_present = w.left_present;
  a.b = BoundTab{a.b.row, w.end, w.prio, w.start, w.gid, w.flags, w.idx, w.req, w.suf, w.suf_online, w.suf_bad,
                 w.suf_vio, Vp};
  a.pp = w_pp.as<PreemptPod>();
  if (hp) {   // the live masks: the bound ones start as the node side's, the nominated ones empty
    CK(cudaMemcpyAsync(h_conf.p, q.conf.data(), (size_t)n * 8, cudaMemcpyHostToDevice, e->s));
    CK(cudaMemcpyAsync(h_want.p, q.want.data(), (size_t)n * 8, cudaMemcpyHostToDevice, e->s));
    CK(dup(h_used, e->hp.d_used.p, (size_t)Npad * 8));
    CK(cudaMemsetAsync(h_nom.p, 0, (size_t)Npad * 8, e->s));
    CK(dup(h_ports, e->hp.d_bports.p, (size_t)Vp * 8));
    CK(dup(h_suf, e->hp.d_bsuf.p, (size_t)Vp * 8));
    hw.used = h_used.as<uint64_t>();
    hw.nom = h_nom.as<uint64_t>();
    hw.ports = h_ports.as<uint64_t>();
    hw.suf_ports = h_suf.as<uint64_t>();
    if (gang) {
      hw.ent_used = he_used.as<uint64_t>();
      hw.ent_nom = he_nom.as<uint64_t>();
      hw.row_ports = hr_ports.as<uint64_t>();
    }
    hp_views(ha, hw.used, hw.nom, hw.ports, hw.suf_ports, h_conf.as<uint64_t>(), h_want.as<uint64_t>());
  }
  a.tiles = w_tiles.as<PickKey>();
  a.out_node = w_node.as<int32_t>();
  a.out_nv = w_nv.as<uint32_t>();
  a.out_cand = w_cand.as<uint32_t>();
  a.victims = w_vict.as<uint32_t>();
  for (uint32_t i = 0; i < n; ++i) {   // stream-ordered: no host synchronisation inside the walk
    with_preempt_build(L, hp, [&](auto M, auto H) {
      if (N) {
        a.p0 = i;
        preempt_node_kernel<M, H><<<dim3(a.n_tiles, 1), PREEMPT_THREADS, 0, e->s>>>(PreemptArgsOf<H>(ha));
        ++e->launches;
      }
      preempt_commit_kernel<M, H><<<1, PREEMPT_THREADS, 0, e->s>>>(PreemptArgsOf<H>(ha), WalkArgsOf<H>(hw), i);
      ++e->launches;
    });
  }
  return preempt_read_back(e, "bs_preempt_walk", a, n, out, [&]() -> int {
    if (outcome) CK(cudaMemcpyAsync(outcome, w.outcome, (size_t)n * 4, cudaMemcpyDeviceToHost, e->s));
    if (evicted_by && V) CK(cudaMemcpyAsync(evicted_by, w.evicted_by, (size_t)V * 4, cudaMemcpyDeviceToHost, e->s));
    return BS_OK;
  }, [](uint64_t) { return BS_OK; });
}

// core.PreemptRemovePod (core.go:203-260).  "Offline" = carries the group label (VerifyPodLabelSatisfied,
// k8s.go:62-70): gid >= 0 or BS_GID_MISSING.  The same-group test (:251) compares fullNameToRemove, which is "" when
// checkPreemption failed, so a victim of p's own group whose group is locked reports the phase message.
int bs_remove_pod(bs_engine* e, uint32_t pod, uint32_t bound, bs_status* st) {
  if (!e || !st) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->have_pods || !e->have_groups || !e->have_bound)
    return fail(e, BS_E_STATE, "bs_remove_pod: upload groups, pods and the bound-pod table first");
  if (pod >= e->P || bound >= e->V) return fail(e, BS_E_INDEX, "bs_remove_pod: index out of range");
  const int32_t gp = e->h_gid[pod], gv = e->h_bgid[bound];
  if (gv >= (int32_t)e->G) return fail(e, BS_E_INDEX, "bs_remove_pod: the bound pod's group index >= n_groups");
  const bool off_p = gp != BS_GID_NONE, off_v = gv != BS_GID_NONE;
  int reason = BS_REMOVE_ALLOW;
  if (!off_p && !off_v) reason = BS_REMOVE_ALLOW;                               // :213-215
  else if (off_p && !off_v) reason = BS_REMOVE_OFFLINE_ONLINE;                  // :216-218
  else {
    int check = BS_REMOVE_ALLOW;                                                // checkPreemption :220-240
    if (gv < 0) check = BS_REMOVE_NOT_FOUND;                                    // :222-225
    else if (e->h_bflags[bound] & BS_BOUND_GROUP_LOCKED) check = BS_REMOVE_LOCKED;   // :234-238
    if (!off_p) reason = check;                                                 // :245-247
    else if (check == BS_REMOVE_ALLOW && gp >= 0 && gp == gv) reason = BS_REMOVE_SAME_GROUP;   // :250-253
    else reason = check;                                                        // :254-256
  }
  st->reason = reason;
  st->code = reason == BS_REMOVE_ALLOW ? BS_CODE_SUCCESS : BS_CODE_UNSCHEDULABLE;   // batchscheduler.go:137-143
  st->group = off_v && gv >= 0 ? gv : -1;
  return BS_OK;
}

int bs_format_remove_message(const bs_status* st, const char* pod_name, const char* victim_name,
                             const char* victim_ns_name, char* buf, size_t buf_len) {
  if (!st || !buf || !buf_len) return BS_E_INVAL;
  std::string m;
  switch (st->reason) {
    case BS_REMOVE_ALLOW: break;
    case BS_REMOVE_OFFLINE_ONLINE:
      m = std::string("offline pods ") + (pod_name ? pod_name : "") + " are forbidden to preempt online " +
          (victim_name ? victim_name : "");
      break;
    case BS_REMOVE_NOT_FOUND: m = std::string("can not found pod group: ") + (victim_ns_name ? victim_ns_name : ""); break;
    case BS_REMOVE_LOCKED: m = "pod belongs to Scheduled or Running pod group can not be scheduled"; break;
    case BS_REMOVE_SAME_GROUP: m = "podToSchedule and podToRemove belong to same pod group, do not preempt"; break;
    default: return BS_E_INVAL;
  }
  if (m.size() + 1 > buf_len) return BS_E_INVAL;
  memcpy(buf, m.c_str(), m.size() + 1);
  return BS_OK;
}

int bs_device_buffer(bs_engine* e, int which, void** dev_ptr, size_t* bytes) {
  if (!e || !dev_ptr || !bytes) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  const uint32_t P = e->P, G = e->G;
  switch (which) {
    case BS_BUF_FIT_BITMAP: *dev_ptr = e->d_fit_bitmap.p; *bytes = (size_t)P * e->bitmap_pitch * 4; break;   // rows of bs_bitmap_pitch words
    case BS_BUF_SCORE: *dev_ptr = e->d_score.p; *bytes = (size_t)P * e->score_pitch * 8; break;   // rows of bs_score_pitch elements
    case BS_BUF_ADMIT_BITMAP: *dev_ptr = e->d_admit_bitmap.p; *bytes = (size_t)cdiv(G, 32) * 4; break;
    case BS_BUF_PREFILTER: *dev_ptr = e->d_prefilter.p; *bytes = P; break;
    case BS_BUF_ADMIT: *dev_ptr = e->d_admit.p; *bytes = G; break;
    case BS_BUF_ORDER: *dev_ptr = e->d_order.p; *bytes = (size_t)P * 4; break;
    case BS_BUF_GATHERED_ADMIT:   // the slot set of the last round (they alternate with the parity of the round number)
      *dev_ptr = e->d_gather.p ? e->d_gather.as<uint32_t>() + (size_t)(e->peer_seq & 1u) * e->peer_world * e->peer_wpr : nullptr;
      *bytes = (size_t)e->peer_world * e->peer_wpr * 4;
      break;
    default: return BS_E_INVAL;
  }
  return BS_OK;
}

void* bs_stream(bs_engine* e) { return e ? (void*)e->s : nullptr; }

uint32_t bs_score_pitch(const bs_engine* e) { return e ? e->score_pitch : 0; }
uint32_t bs_bitmap_pitch(const bs_engine* e) { return e ? e->bitmap_pitch : 0; }

int bs_fetch_fit_rows(bs_engine* e, uint32_t pod0, uint32_t n, uint32_t* words) {
  if (!e || !words) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->evaluated || !(e->out_flags & BS_OUT_FIT_BITMAP)) return fail(e, BS_E_STATE, "no fit bitmap materialised");
  if ((uint64_t)pod0 + n > e->P) return BS_E_INDEX;
  BS_DEVICE_GUARD(e);
  if (n && e->W)
    CK(cudaMemcpy2DAsync(words, (size_t)e->W * 4, e->d_fit_bitmap.as<uint32_t>() + (size_t)pod0 * e->bitmap_pitch,
                         (size_t)e->bitmap_pitch * 4, (size_t)e->W * 4, n, cudaMemcpyDeviceToHost, e->s));
  CK(cudaStreamSynchronize(e->s));
  return BS_OK;
}

int bs_fetch_filter_rows(bs_engine* e, uint32_t pod0, uint32_t n, uint32_t* words) {
  if (!e || !words) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->evaluated || !(e->out_flags & BS_OUT_FILTER)) return fail(e, BS_E_STATE, "no filter matrix materialised");
  if ((uint64_t)pod0 + n > e->P) return BS_E_INDEX;
  BS_DEVICE_GUARD(e);
  if (n && e->W)
    CK(cudaMemcpyAsync(words, e->d_filter_bitmap.as<uint32_t>() + (size_t)pod0 * e->W, (size_t)n * e->W * 4,
                       cudaMemcpyDeviceToHost, e->s));
  CK(cudaStreamSynchronize(e->s));
  return BS_OK;
}

int bs_filter(bs_engine* e, uint32_t pod, uint32_t node, bs_status* st) {
  if (!e || !st) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->evaluated || !(e->out_flags & BS_OUT_FILTER)) return fail(e, BS_E_STATE, "bs_filter: evaluate with BS_OUT_FILTER first");
  if (pod >= e->P || node >= e->N) return BS_E_INDEX;
  if (!e->fetched) {
    int rc = fetch_locked(e, nullptr);
    if (rc) return rc;
  }
  BS_DEVICE_GUARD(e);
  uint32_t word = 0;
  const uint8_t nflag = e->h_nflags[node];
  CK(cudaMemcpyAsync(&word, e->d_filter_bitmap.as<uint32_t>() + (size_t)pod * e->W + (node >> 5), 4,
                     cudaMemcpyDeviceToHost, e->s));
  CK(cudaStreamSynchronize(e->s));
  const int32_t g = e->h_gid[pod];
  st->group = (g >= 0 && (uint32_t)g < e->G) ? g : -1;
  const uint8_t pcode = e->h_filter_code.as<uint8_t>()[pod];
  if ((word >> (node & 31)) & 1u) st->reason = BS_FILTER_PASS;
  else if (pcode != BS_FILTER_PASS) st->reason = pcode;
  else st->reason = (nflag & BS_NODE_NIL) ? BS_FILTER_ERR_NO_SNAPSHOT : BS_FILTER_ERR_NOT_ENOUGH;
  st->code = st->reason == BS_FILTER_PASS ? BS_CODE_SUCCESS : BS_CODE_UNSCHEDULABLE;   // batchscheduler.go:153-156
  return BS_OK;
}

int bs_fetch_score_rows(bs_engine* e, uint32_t pod0, uint32_t n, int64_t* scores) {
  if (!e || !scores) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->evaluated || !(e->out_flags & BS_OUT_SCORE)) return fail(e, BS_E_STATE, "no score matrix materialised");
  if ((uint64_t)pod0 + n > e->P) return BS_E_INDEX;
  BS_DEVICE_GUARD(e);
  if (n && e->N)
    CK(cudaMemcpy2DAsync(scores, (size_t)e->N * 8, e->d_score.as<int64_t>() + (size_t)pod0 * e->score_pitch,
                         (size_t)e->score_pitch * 8, (size_t)e->N * 8, n, cudaMemcpyDeviceToHost, e->s));
  CK(cudaStreamSynchronize(e->s));
  return BS_OK;
}

int bs_fetch_topk_rows(bs_engine* e, uint32_t pod0, uint32_t n, int32_t* nodes, int64_t* scores) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->evaluated || !(e->out_flags & BS_OUT_TOPK)) return fail(e, BS_E_STATE, "no top-K lists materialised");
  if ((uint64_t)pod0 + n > e->P) return BS_E_INDEX;
  BS_DEVICE_GUARD(e);
  const size_t off = (size_t)pod0 * e->topk, cnt = (size_t)n * e->topk;   // device rows are dense [Prows][K]
  if (cnt && nodes)
    CK(cudaMemcpyAsync(nodes, e->d_topk_node.as<int32_t>() + off, cnt * 4, cudaMemcpyDeviceToHost, e->s));
  if (cnt && scores)
    CK(cudaMemcpyAsync(scores, e->d_topk_score.as<int64_t>() + off, cnt * 8, cudaMemcpyDeviceToHost, e->s));
  CK(cudaStreamSynchronize(e->s));
  return BS_OK;
}

int bs_fetch_reason_rows(bs_engine* e, uint32_t pod0, uint32_t n, uint32_t* counts) {
  if (!e || !counts) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->evaluated || !(e->out_flags & BS_OUT_REASONS)) return fail(e, BS_E_STATE, "no reason rows materialised");
  if ((uint64_t)pod0 + n > e->P) return BS_E_INDEX;
  BS_DEVICE_GUARD(e);
  const size_t R = 4 + e->L;
  if (n) CK(cudaMemcpyAsync(counts, e->d_reasons.as<uint32_t>() + (size_t)pod0 * R, (size_t)n * R * 4,
                            cudaMemcpyDeviceToHost, e->s));
  CK(cudaStreamSynchronize(e->s));
  return BS_OK;
}

// ---- resource priorities (BS_OUT_PRIORITY, priority.cuh) ----
int bs_set_score_weights(bs_engine* e, uint32_t least, uint32_t most, uint32_t balanced) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  e->weights = ScoreWeights{least, most, balanced};
  return BS_OK;
}

int bs_set_ratio_priority(bs_engine* e, uint32_t weight, uint32_t n_points, const uint32_t* utilization,
                          const uint32_t* score, uint32_t n_lanes, const uint32_t* lane_weight, uint32_t absent_weight) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  const char* who = "bs_set_ratio_priority";
  auto bad = [&](const char* why) { return fail(e, BS_E_INVAL, (std::string(who) + ": " + why).c_str()); };
  if (n_points < 1 || n_points > (uint32_t)RATIO_TABLE) return bad("the shape needs 1 to 101 points");
  if (!utilization || !score || !lane_weight) return bad("null argument");
  for (uint32_t i = 0; i < n_points; ++i) {
    if (utilization[i] > 100 || score[i] > 100) return bad("utilization and score lie in [0, 100]");
    if (i && utilization[i] <= utilization[i - 1]) return bad("utilization must be strictly ascending");
  }
  if (n_lanes != e->L) return bad("n_lanes differs from the engine's");
  if (lane_weight[LANE_PODS]) return bad("lane 3 (pods) must weigh 0: pass its weight in absent_weight");
  uint64_t sum = absent_weight;
  for (uint32_t d = 0; d < n_lanes; ++d) sum += lane_weight[d];
  if (sum > (1u << 24)) return bad("the weights sum to more than 2^24");
  // buildBrokenLinearFunction [upstream, from memory] at every utilization 0..100, int64 truncating toward zero
  int32_t tab[RATIO_TABLE];
  for (int64_t p = 0; p < RATIO_TABLE; ++p) {
    int64_t v = score[n_points - 1];
    for (uint32_t i = 0; i < n_points; ++i) {
      if (p > (int64_t)utilization[i]) continue;
      if (i == 0) v = score[0];
      else {
        const int64_t s0 = score[i - 1], s1 = score[i], u0 = utilization[i - 1], u1 = utilization[i];
        v = s0 + (s1 - s0) * (p - u0) / (u1 - u0);
      }
      break;
    }
    tab[p] = (int32_t)v;
  }
  BS_DEVICE_GUARD(e);
  CK(e->d_ratio_tab.ensure(sizeof tab));
  CK(cudaMemcpyAsync(e->d_ratio_tab.p, tab, sizeof tab, cudaMemcpyHostToDevice, e->s));
  CK(cudaStreamSynchronize(e->s));
  RatioSetting r{};
  r.table = e->d_ratio_tab.as<int32_t>();
  for (uint32_t d = 0; d < n_lanes; ++d) {
    r.lane_w[d] = lane_weight[d];
    if (lane_weight[d]) r.mask |= 1u << d;
  }
  r.weight = weight;
  if (tab[100] > 0) { r.num0 = (uint32_t)tab[100] * absent_weight; r.den0 = absent_weight; }
  e->ratio = r;
  return BS_OK;
}

namespace {
// One non-zero column [2][n] (the node or the pod half) into its device column ([2][pitch], zero beyond n), marked
// present only when every value lies in [0, BS_NONZERO_MAX].  Its maxima go to node_max / pod_max
// (bs_replay_priority's overflow bound).
int upload_nonzero(bs_engine* e, SideOf side, uint32_t n, const int64_t* nz) {
  const bool node = side == NODE_SIDE;
  const Refuse bad{e, node ? "bs_upload_node_nonzero" : "bs_upload_pod_nonzero"};
  bool& have = node ? e->nz.have_node : e->nz.have_pod;
  int64_t(&mx)[2] = node ? e->nz.node_max : e->nz.pod_max;
  have = false;
  if (int rc = bad.shape(side, n)) return rc;
  if (n && !nz) return bad(BS_E_INVAL, "null column");
  mx[0] = mx[1] = 0;
  for (size_t k = 0; k < (size_t)2 * n; ++k) {
    if (nz[k] < 0 || nz[k] > BS_NONZERO_MAX) return fail(e, BS_E_RANGE, "non-zero request outside [0, 2^56]");
    int64_t& m = mx[k >= n];
    m = std::max(m, nz[k]);
  }
  BS_DEVICE_GUARD(e);
  if (int rc = upload_col(e, col(nz, node ? e->nz.d_node : e->nz.d_pod, 2), n, node ? e->Npad : n)) return rc;
  CK(cudaStreamSynchronize(e->s));
  have = true;
  return BS_OK;
}
}  // namespace

int bs_upload_node_nonzero(bs_engine* e, uint32_t n_nodes, const int64_t* nz) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  return upload_nonzero(e, NODE_SIDE, n_nodes, nz);
}

int bs_upload_pod_nonzero(bs_engine* e, uint32_t n_pods, const int64_t* nz) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  return upload_nonzero(e, POD_SIDE, n_pods, nz);
}

int bs_set_node_priority_weights(bs_engine* e, uint32_t taint_toleration, uint32_t node_affinity) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  e->w_taint = taint_toleration;
  e->w_naff = node_affinity;
  return BS_OK;
}

int bs_upload_node_preferences(bs_engine* e, uint32_t n_nodes, const uint64_t* prefer_taints, uint32_t n_classes,
                               const int32_t* pref_weights) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  const Refuse bad{e, "bs_upload_node_preferences"};
  e->pref.have_node = false;
  if (int rc = bad.shape(NODE_SIDE, n_nodes)) return rc;
  const uint32_t Npad = e->Npad;
  if ((uint64_t)n_classes * Npad * 4 > BS_PREF_TABLE_MAX_BYTES)
    return bad(BS_E_INVAL, "n_classes x padded nodes x 4 bytes exceeds BS_PREF_TABLE_MAX_BYTES");
  if (n_nodes && !prefer_taints) return bad(BS_E_INVAL, "null prefer_taints");
  if (n_classes && n_nodes && !pref_weights) return bad(BS_E_INVAL, "null pref_weights");
  for (size_t k = 0; k < (size_t)n_classes * n_nodes; ++k)
    if (pref_weights[k] < 0) return bad(BS_E_RANGE, "a preferred-affinity weight is negative");
  BS_DEVICE_GUARD(e);
  int rc;
  if ((rc = upload_vec(e, e->pref.d_prefer_taints, prefer_taints, n_nodes, Npad))) return rc;
  if (n_classes && (rc = upload_col(e, col(pref_weights, e->pref.d_weights, n_classes), n_nodes, Npad))) return rc;
  CK(cudaStreamSynchronize(e->s));
  e->pref.classes = n_classes;
  e->pref.have_node = true;
  return BS_OK;
}

int bs_upload_pod_preferences(bs_engine* e, uint32_t n_pods, const uint64_t* prefer_tol, const uint32_t* pref_class) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  const Refuse bad{e, "bs_upload_pod_preferences"};
  e->pref.have_pod = false;
  if (int rc = bad.shape(POD_SIDE, n_pods)) return rc;
  if (n_pods && (!prefer_tol || !pref_class)) return bad(BS_E_INVAL, "null column");
  const int64_t mx = max_class(pref_class, n_pods, BS_PREF_NONE);
  BS_DEVICE_GUARD(e);
  int rc;
  if ((rc = upload_vec(e, e->pref.d_prefer_tol, prefer_tol, n_pods, n_pods))) return rc;
  if ((rc = upload_vec(e, e->pref.d_class, pref_class, n_pods, n_pods))) return rc;
  CK(cudaStreamSynchronize(e->s));
  e->pref.class_max = mx;
  e->pref.have_pod = true;
  return BS_OK;
}

int bs_set_locality_weights(bs_engine* e, uint32_t image_locality, uint32_t prefer_avoid_pods) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  if (image_locality != e->w_img || prefer_avoid_pods != e->w_avoid) e->loc.dirty = true;
  e->w_img = image_locality;
  e->w_avoid = prefer_avoid_pods;
  return BS_OK;
}

int bs_upload_node_locality(bs_engine* e, uint32_t n_nodes, uint32_t n_images, const int64_t* image_size,
                            const uint32_t* image_bits, const uint64_t* avoid_mask) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  const Refuse bad{e, "bs_upload_node_locality"};
  e->loc.have_img_node = e->loc.have_avoid_node = false;
  e->loc.dirty = true;
  if (int rc = bad.shape(NODE_SIDE, n_nodes)) return rc;
  const uint32_t Npad = e->Npad, words = cdiv(n_nodes, 32);
  const bool img = image_size && image_bits;
  if (img && (uint64_t)n_images * words * 4 > BS_LOC_TABLE_MAX_BYTES)
    return bad(BS_E_INVAL, "n_images x ceil(n_nodes / 32) x 4 bytes exceeds BS_LOC_TABLE_MAX_BYTES");
  for (uint32_t i = 0; img && i < n_images; ++i)
    if (image_size[i] < 0 || image_size[i] > BS_IMAGE_SIZE_MAX) return bad(BS_E_RANGE, "an image size is outside [0, 2^48]");
  BS_DEVICE_GUARD(e);
  int rc;
  if (img && (rc = upload_vec(e, e->loc.d_img_size, image_size, n_images, n_images))) return rc;
  const uint64_t bits = (uint64_t)n_images * words;
  if (img && (rc = upload_vec(e, e->loc.d_img_bits, image_bits, bits, bits))) return rc;
  if (avoid_mask && (rc = upload_vec(e, e->loc.d_avoid_mask, avoid_mask, n_nodes, Npad))) return rc;
  CK(cudaStreamSynchronize(e->s));
  e->loc.images = img ? n_images : 0;
  e->loc.have_img_node = img;
  e->loc.have_avoid_node = avoid_mask != nullptr;
  return BS_OK;
}

int bs_upload_pod_locality(bs_engine* e, uint32_t n_pods, const uint32_t* image_class, uint32_t n_classes,
                           const uint32_t* class_offset, const uint32_t* class_images, const uint8_t* avoid_bit) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  const Refuse bad{e, "bs_upload_pod_locality"};
  e->loc.have_img_pod = e->loc.have_avoid_pod = false;
  e->loc.dirty = true;
  if (int rc = bad.shape(POD_SIDE, n_pods)) return rc;
  const bool img = image_class && class_offset && class_images;
  int64_t cmax = -1, imax = -1;
  uint32_t nnz = 0;
  if (img) {
    if ((uint64_t)n_classes * e->Npad > BS_LOC_TABLE_MAX_BYTES)
      return bad(BS_E_INVAL, "n_classes x padded nodes bytes exceeds BS_LOC_TABLE_MAX_BYTES");
    if (class_offset[0] != 0) return bad(BS_E_INVAL, "class_offset[0] is not 0");
    for (uint32_t c = 0; c < n_classes; ++c)
      if (class_offset[c + 1] < class_offset[c] || class_offset[c + 1] - class_offset[c] > BS_LOC_CLASS_MAX)
        return bad(BS_E_INVAL, "class_offset is not ascending, or a class lists more than BS_LOC_CLASS_MAX ids");
    nnz = class_offset[n_classes];
    for (uint32_t k = 0; k < nnz; ++k) imax = std::max(imax, (int64_t)class_images[k]);
    cmax = max_class(image_class, n_pods, BS_IMAGE_NONE);
  }
  for (uint32_t p = 0; avoid_bit && p < n_pods; ++p)
    if (avoid_bit[p] > 63 && avoid_bit[p] != BS_AVOID_NONE) return bad(BS_E_RANGE, "an avoid bit is outside 0..63");
  BS_DEVICE_GUARD(e);
  int rc;
  if (img && ((rc = upload_vec(e, e->loc.d_class, image_class, n_pods, n_pods)) ||
              (rc = upload_vec(e, e->loc.d_off, class_offset, n_classes + 1, n_classes + 1)) ||
              (rc = upload_vec(e, e->loc.d_ids, class_images, nnz, nnz))))
    return rc;
  if (avoid_bit && (rc = upload_vec(e, e->loc.d_avoid_bit, avoid_bit, n_pods, n_pods))) return rc;
  CK(cudaStreamSynchronize(e->s));
  e->loc.classes = img ? n_classes : 0;
  e->loc.class_max = cmax;
  e->loc.image_max = imax;
  e->loc.have_img_pod = img;
  e->loc.have_avoid_pod = avoid_bit != nullptr;
  return BS_OK;
}

int bs_set_spread_weight(bs_engine* e, uint32_t selector_spread) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  e->w_spread = selector_spread;
  return BS_OK;
}

int bs_upload_node_spread(bs_engine* e, uint32_t n_nodes, uint32_t n_zones, const uint8_t* zone, uint32_t n_classes,
                          const int32_t* counts) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  const Refuse bad{e, "bs_upload_node_spread"};
  e->spread.have_node = false;
  if (int rc = bad.shape(NODE_SIDE, n_nodes)) return rc;
  if (n_zones > BS_SPREAD_ZONE_MAX) return bad(BS_E_INVAL, "n_zones exceeds BS_SPREAD_ZONE_MAX");
  const uint32_t Npad = e->Npad;
  if ((uint64_t)n_classes * Npad * 4 > BS_SPREAD_TABLE_MAX_BYTES)
    return bad(BS_E_INVAL, "n_classes x padded nodes x 4 bytes exceeds BS_SPREAD_TABLE_MAX_BYTES");
  if (n_nodes && !zone) return bad(BS_E_INVAL, "null zone");
  if (n_classes && n_nodes && !counts) return bad(BS_E_INVAL, "null counts");
  for (uint32_t i = 0; i < n_nodes; ++i)
    if (zone[i] >= n_zones && zone[i] != BS_ZONE_NONE) return bad(BS_E_INDEX, "a zone id is >= n_zones");
  for (size_t k = 0; k < (size_t)n_classes * n_nodes; ++k)
    if (counts[k] < 0 || counts[k] > BS_SPREAD_COUNT_MAX) return bad(BS_E_RANGE, "a count is outside [0, 2^24]");
  BS_DEVICE_GUARD(e);
  int rc;
  // padding nodes have no zone (and never fit)
  if ((rc = upload_vec(e, e->spread.d_zone, zone, n_nodes, Npad, BS_ZONE_NONE))) return rc;
  if (n_classes && (rc = upload_col(e, col(counts, e->spread.d_counts, n_classes), n_nodes, Npad))) return rc;
  CK(cudaStreamSynchronize(e->s));
  e->spread.classes = n_classes;
  e->spread.have_node = true;
  return BS_OK;
}

int bs_upload_pod_spread(bs_engine* e, uint32_t n_pods, const uint32_t* spread_class) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  const Refuse bad{e, "bs_upload_pod_spread"};
  e->spread.have_pod = false;
  if (int rc = bad.shape(POD_SIDE, n_pods)) return rc;
  if (n_pods && !spread_class) return bad(BS_E_INVAL, "null spread_class");
  const int64_t mx = max_class(spread_class, n_pods, BS_SPREAD_NONE);
  BS_DEVICE_GUARD(e);
  if (int rc = upload_vec(e, e->spread.d_class, spread_class, n_pods, n_pods)) return rc;
  CK(cudaStreamSynchronize(e->s));
  e->spread.class_max = mx;
  e->spread.have_pod = true;
  return BS_OK;
}

int bs_set_interpod_weight(bs_engine* e, uint32_t inter_pod_affinity) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  e->w_ipa = inter_pod_affinity;
  return BS_OK;
}

namespace {

// A class table of bs_interpod_classes: the offsets ascending from 0 and at most BS_IPA_CLASS_MAX apart, own and match
// in range, the terms distinct within a class and (n_terms != UINT32_MAX) below n_terms.  term_max: the largest term.
int interpod_classes_check(const bs_interpod_classes& c, uint32_t n_terms, int64_t& term_max, const char*& why) {
  term_max = -1;
  if (!c.n_classes) return BS_OK;
  if (!c.class_offset) return why = "null class_offset", BS_E_INVAL;
  if (c.class_offset[0] != 0) return why = "class_offset[0] is not 0", BS_E_INVAL;
  for (uint32_t k = 0; k < c.n_classes; ++k)
    if (c.class_offset[k + 1] < c.class_offset[k] || c.class_offset[k + 1] - c.class_offset[k] > BS_IPA_CLASS_MAX)
      return why = "class_offset is not ascending, or a class lists more than BS_IPA_CLASS_MAX entries", BS_E_INVAL;
  const uint32_t nnz = c.class_offset[c.n_classes];
  if (nnz && !(c.term && c.own && c.match)) return why = "null term, own or match", BS_E_INVAL;
  for (uint32_t k = 0; k < nnz; ++k) {
    if (c.match[k] > 1) return why = "a match is not 0 or 1", BS_E_RANGE;
    if (c.own[k] < -BS_IPA_OWN_MAX || c.own[k] > BS_IPA_OWN_MAX) return why = "an own is outside [-2^16, 2^16]", BS_E_RANGE;
    if (n_terms != UINT32_MAX && c.term[k] >= n_terms) return why = "a term id is >= n_terms", BS_E_INDEX;
    term_max = std::max(term_max, (int64_t)c.term[k]);
  }
  for (uint32_t k = 0; k < c.n_classes; ++k) {
    const uint32_t o0 = c.class_offset[k], o1 = c.class_offset[k + 1];
    for (uint32_t x = o0; x < o1; ++x)
      for (uint32_t y = x + 1; y < o1; ++y)
        if (c.term[x] == c.term[y]) return why = "a class lists one term twice", BS_E_INVAL;
  }
  return BS_OK;
}

// Device copies of a checked class table (an offset 0 alone for an empty one).
int interpod_classes_upload(bs_engine* e, const bs_interpod_classes& c, DevBuf& off, DevBuf& term, DevBuf& own,
                            DevBuf& match) {
  const uint32_t nnz = c.n_classes ? c.class_offset[c.n_classes] : 0;
  int rc;
  if ((rc = upload_vec(e, off, c.class_offset, c.n_classes ? c.n_classes + 1 : 0, c.n_classes + 1)) ||
      (rc = upload_vec(e, term, c.term, nnz, nnz)) || (rc = upload_vec(e, own, c.own, nnz, nnz)) ||
      (rc = upload_vec(e, match, c.match, nnz, nnz)))
    return rc;
  return BS_OK;
}

// What the node sides of InterPodAffinity and of the MatchInterPodAffinity filter differ in.
struct InterpodLimits {
  uint32_t bound_max;   // bound pods at most
  uint32_t none;        // the class of a bound pod without entries
  bool planes;          // the slots are the filter's two presence bit planes, not the priority's 16-byte M and S
  bool own_01;          // every own is 0 or 1 (the filter's anti-affinity flag)
  const char *bound_why, *slots_why;
};
constexpr InterpodLimits IPA_LIMITS{BS_IPA_BOUND_MAX, BS_IPA_NONE, false, false, "n_bound exceeds BS_IPA_BOUND_MAX",
                                    "the term tables exceed BS_IPA_TERM_MAX_BYTES"};
constexpr InterpodLimits IPF_LIMITS{BS_IPF_BOUND_MAX, BS_IPF_NONE, true, true, "n_bound exceeds BS_IPF_BOUND_MAX",
                                    "the presence planes exceed BS_IPF_TERM_MAX_BYTES"};

// Checks a bs_interpod_nodes table against the node table and `lim`, and copies it into s.  The caller has dropped
// the side already.
int upload_interpod_nodes(bs_engine* e, const Refuse& bad, const bs_interpod_nodes* t, const InterpodLimits& lim,
                          InterpodNodeSide& s) {
  if (!t) return bad(BS_E_INVAL, "null table");
  if (int rc = bad.shape(NODE_SIDE, t->n_nodes)) return rc;
  const uint32_t N = t->n_nodes, K = t->n_keys, T = t->n_terms, V = t->n_bound;
  if (K > BS_IPA_KEY_MAX) return bad(BS_E_INVAL, "n_keys exceeds BS_IPA_KEY_MAX");
  if (V > lim.bound_max) return bad(BS_E_INVAL, lim.bound_why);
  if ((K && !t->n_values) || (K && N && !t->topo) || (T && !t->term_key) || (V && !(t->bound_node && t->bound_class)))
    return bad(BS_E_INVAL, "null column");
  for (size_t k = 0; k < (size_t)K * N; ++k)
    if (t->topo[k] != BS_TOPO_NONE && t->topo[k] >= t->n_values[k / N]) return bad(BS_E_INDEX, "a topo value is >= n_values");
  std::vector<uint32_t> off(T);
  uint64_t slots = 0;
  for (uint32_t k = 0; k < T; ++k) {
    if (t->term_key[k] >= K) return bad(BS_E_INDEX, "a term_key is >= n_keys");
    off[k] = lim.planes ? (uint32_t)slots : (uint32_t)std::min<uint64_t>(slots, UINT32_MAX);
    slots += t->n_values[t->term_key[k]];
    if (lim.planes ? (slots + 31) / 32 * 2 * 4 > BS_IPF_TERM_MAX_BYTES : slots * 16 > BS_IPA_TERM_MAX_BYTES)
      return bad(BS_E_INVAL, lim.slots_why);
  }
  for (uint32_t k = 0; k < V; ++k) {
    if (t->bound_node[k] >= N) return bad(BS_E_INDEX, "a bound_node is >= n_nodes");
    if (t->bound_class[k] != lim.none && t->bound_class[k] >= t->classes.n_classes)
      return bad(BS_E_INDEX, "a bound_class is >= n_classes");
  }
  int64_t tmax;
  const char* why = nullptr;
  if (int rc = interpod_classes_check(t->classes, T, tmax, why)) return bad(rc, why);
  const uint32_t nnz = t->classes.n_classes ? t->classes.class_offset[t->classes.n_classes] : 0;
  for (uint32_t k = 0; lim.own_01 && k < nnz; ++k)
    if (t->classes.own[k] != 0 && t->classes.own[k] != 1) return bad(BS_E_RANGE, "an own is not 0 or 1");
  BS_DEVICE_GUARD(e);
  const uint64_t KN = (uint64_t)K * N;
  int rc;
  if ((rc = upload_vec(e, s.d_topo, t->topo, KN, KN)) || (rc = upload_vec(e, s.d_term_key, t->term_key, T, T)) ||
      (rc = upload_vec(e, s.d_term_off, off.data(), T, T)) ||
      (rc = upload_vec(e, s.d_bound_node, t->bound_node, V, V)) ||
      (rc = upload_vec(e, s.d_bound_class, t->bound_class, V, V)) ||
      (rc = interpod_classes_upload(e, t->classes, s.d_boff, s.d_bterm, s.d_bown, s.d_bmatch)))
    return rc;
  CK(cudaStreamSynchronize(e->s));   // the caller's columns may go once the call returns
  s.terms = T;
  s.slots = slots;
  s.bound = V;
  s.bclasses = t->classes.n_classes;
  return BS_OK;
}

}  // namespace

int bs_upload_node_interpod(bs_engine* e, const bs_interpod_nodes* t) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  e->ipa.have_node = false;
  e->ipa.dirty = e->ipa.mass_dirty = true;
  const int rc = upload_interpod_nodes(e, {e, "bs_upload_node_interpod"}, t, IPA_LIMITS, e->ipa.node);
  e->ipa.have_node = rc == BS_OK;
  return rc;
}

int bs_upload_pod_interpod(bs_engine* e, const bs_interpod_pods* t) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  const Refuse bad{e, "bs_upload_pod_interpod"};
  e->ipa.have_pod = false;
  e->ipa.dirty = true;
  if (!t) return bad(BS_E_INVAL, "null table");
  const uint32_t P = t->n_pods;
  if (int rc = bad.shape(POD_SIDE, P)) return rc;
  if (P && !t->pod_class) return bad(BS_E_INVAL, "null pod_class");
  if ((uint64_t)t->classes.n_classes * e->Npad * 8 > BS_IPA_TABLE_MAX_BYTES)
    return bad(BS_E_INVAL, "n_classes x padded nodes x 8 bytes exceeds BS_IPA_TABLE_MAX_BYTES");
  if (max_class(t->pod_class, P, BS_IPA_NONE) >= (int64_t)t->classes.n_classes)
    return bad(BS_E_INDEX, "a pod_class is >= n_classes");
  int64_t tmax;
  const char* why = nullptr;
  if (int rc = interpod_classes_check(t->classes, UINT32_MAX, tmax, why)) return bad(rc, why);
  BS_DEVICE_GUARD(e);
  int rc;
  if ((rc = upload_vec(e, e->ipa.d_class, t->pod_class, P, P)) ||
      (rc = interpod_classes_upload(e, t->classes, e->ipa.d_poff, e->ipa.d_pterm, e->ipa.d_pown, e->ipa.d_pmatch)))
    return rc;
  CK(cudaStreamSynchronize(e->s));
  e->ipa.pclasses = t->classes.n_classes;
  e->ipa.term_max = tmax;
  e->ipa.have_pod = true;
  return BS_OK;
}

int bs_set_interpod_filter(bs_engine* e, int on) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  if ((on != 0) == e->ipf.on) return BS_OK;
  e->ipf.on = on != 0;
  e->ipf.dirty = true;   // the pass bits are built again at the next evaluation the filter is on for
  e->filt.assign_dirty = e->classes_dirty = e->pod_classes_dirty = true;   // and the pods' fit classes follow the switch
  e->evaluated = false;
  return BS_OK;
}

int bs_upload_node_interpod_filter(bs_engine* e, const bs_interpod_nodes* t) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  e->ipf.have_node = false;
  e->ipf.dirty = true;
  const int rc = upload_interpod_nodes(e, {e, "bs_upload_node_interpod_filter"}, t, IPF_LIMITS, e->ipf.node);
  if (rc) return rc;
  e->ipf.have_node = true;
  e->evaluated = false;
  return BS_OK;
}

int bs_upload_pod_interpod_filter(bs_engine* e, const bs_interpod_filter_pods* t) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  const Refuse bad{e, "bs_upload_pod_interpod_filter"};
  e->ipf.have_pod = false;
  e->ipf.dirty = true;
  if (!t) return bad(BS_E_INVAL, "null table");
  const uint32_t P = t->n_pods, C = t->n_classes;
  if (int rc = bad.shape(POD_SIDE, P)) return rc;
  if (P && !t->pod_class) return bad(BS_E_INVAL, "null pod_class");
  if (C && !(t->class_offset && t->self_match)) return bad(BS_E_INVAL, "null class_offset or self_match");
  if (3ull * C * (e->Npad / 8) > BS_IPF_TABLE_MAX_BYTES)
    return bad(BS_E_INVAL, "3 x n_classes x padded nodes / 8 bytes exceeds BS_IPF_TABLE_MAX_BYTES");
  if (C && t->class_offset[0] != 0) return bad(BS_E_INVAL, "class_offset[0] is not 0");
  for (uint32_t k = 0; k < C; ++k)
    if (t->class_offset[k + 1] < t->class_offset[k] || t->class_offset[k + 1] - t->class_offset[k] > BS_IPF_CLASS_MAX)
      return bad(BS_E_INVAL, "class_offset is not ascending, or a class lists more than BS_IPF_CLASS_MAX entries");
  const uint32_t nnz = C ? t->class_offset[C] : 0;
  if (nnz && !(t->term && t->role)) return bad(BS_E_INVAL, "null term or role");
  int64_t tmax = -1;
  for (uint32_t k = 0; k < nnz; ++k) {
    if (t->role[k] > BS_IPF_EXISTING) return bad(BS_E_INVAL, "a role is not BS_IPF_AFFINITY, BS_IPF_ANTI or BS_IPF_EXISTING");
    tmax = std::max(tmax, (int64_t)t->term[k]);
  }
  for (uint32_t k = 0; k < C; ++k)
    if (t->self_match[k] > 1) return bad(BS_E_RANGE, "a self_match is not 0 or 1");
  if (max_class(t->pod_class, P, BS_IPF_NONE) >= (int64_t)C) return bad(BS_E_INDEX, "a pod_class is >= n_classes");
  BS_DEVICE_GUARD(e);
  const uint32_t offs = C ? C + 1 : 0;   // (no offset at all for an empty table: no class is ever read)
  int rc;
  if ((rc = upload_vec(e, e->ipf.d_poff, t->class_offset, offs, offs)) ||
      (rc = upload_vec(e, e->ipf.d_pterm, t->term, nnz, nnz)) || (rc = upload_vec(e, e->ipf.d_prole, t->role, nnz, nnz)) ||
      (rc = upload_vec(e, e->ipf.d_pself, t->self_match, C, C)))
    return rc;
  CK(cudaStreamSynchronize(e->s));
  e->ipf.h_class.assign(t->pod_class, t->pod_class + P);
  e->ipf.pclasses = C;
  e->ipf.term_max = tmax;
  e->ipf.have_pod = true;
  e->filt.assign_dirty = e->classes_dirty = e->pod_classes_dirty = true;   // the pods' fit classes carry the filter class
  e->evaluated = false;
  return BS_OK;
}

int bs_upload_pod_interpod_placed(bs_engine* e, const bs_interpod_pods* t) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  const Refuse bad{e, "bs_upload_pod_interpod_placed"};
  e->ipf.have_placed = false;
  if (!t) return bad(BS_E_INVAL, "null table");
  const uint32_t P = t->n_pods;
  if (int rc = bad.shape(POD_SIDE, P)) return rc;
  if (P && !t->pod_class) return bad(BS_E_INVAL, "null pod_class");
  if (max_class(t->pod_class, P, BS_IPF_NONE) >= (int64_t)t->classes.n_classes)
    return bad(BS_E_INDEX, "a pod_class is >= n_classes");
  int64_t tmax;
  const char* why = nullptr;
  if (int rc = interpod_classes_check(t->classes, UINT32_MAX, tmax, why)) return bad(rc, why);
  const uint32_t nnz = t->classes.n_classes ? t->classes.class_offset[t->classes.n_classes] : 0;
  for (uint32_t k = 0; k < nnz; ++k)
    if (t->classes.own[k] != 0 && t->classes.own[k] != 1) return bad(BS_E_RANGE, "an own is not 0 or 1");
  BS_DEVICE_GUARD(e);
  int rc;
  if ((rc = upload_vec(e, e->ipf.d_qclass, t->pod_class, P, P)) ||
      (rc = interpod_classes_upload(e, t->classes, e->ipf.d_qoff, e->ipf.d_qterm, e->ipf.d_qown, e->ipf.d_qmatch)))
    return rc;
  CK(cudaStreamSynchronize(e->s));
  e->ipf.placed_term_max = tmax;
  e->ipf.have_placed = true;
  return BS_OK;
}

int bs_fetch_interpod_reason_rows(bs_engine* e, uint32_t pod0, uint32_t n, uint32_t* counts) {
  if (!e || (n && !counts)) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->evaluated || !(e->out_flags & BS_OUT_REASONS)) return fail(e, BS_E_STATE, "no reason rows materialised");
  if ((uint64_t)pod0 + n > e->P) return BS_E_INDEX;
  if (!n) return BS_OK;
  if (!e->ipf.round) {
    memset(counts, 0, (size_t)n * 3 * 4);
    return BS_OK;
  }
  BS_DEVICE_GUARD(e);
  CK(cudaMemcpyAsync(counts, e->ipf.d_reasons.as<uint32_t>() + (size_t)pod0 * 3, (size_t)n * 3 * 4,
                     cudaMemcpyDeviceToHost, e->s));
  CK(cudaStreamSynchronize(e->s));
  return BS_OK;
}

int bs_set_host_port_filter(bs_engine* e, int on) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  if ((on != 0) == e->hp.on) return BS_OK;
  e->hp.on = on != 0;
  e->hp.dirty = true;   // the class fit bits are built again at the next evaluation the filter is on for
  e->filt.assign_dirty = e->classes_dirty = e->pod_classes_dirty = true;   // and the pods' fit classes follow the switch
  e->evaluated = false;
  return BS_OK;
}

int bs_upload_node_host_ports(bs_engine* e, const bs_host_port_nodes* t) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  const Refuse bad{e, "bs_upload_node_host_ports"};
  e->hp.have_node = false;
  if (!t) return bad(BS_E_INVAL, "null table");
  const uint32_t N = t->n_nodes, K = t->n_entries;
  if (int rc = bad.shape(NODE_SIDE, N)) return rc;
  if (K > BS_HOSTPORT_MAX) return bad(BS_E_INVAL, "more than BS_HOSTPORT_MAX entries");
  if (K && !(t->ip && t->protocol && t->port)) return bad(BS_E_INVAL, "null ip, protocol or port");
  if (N && !t->used) return bad(BS_E_INVAL, "null used");
  for (uint32_t a = 0; a < K; ++a)
    if (t->port[a] < 1 || t->port[a] > 65535) return bad(BS_E_RANGE, "a port is outside 1..65535");
  // entries a and b conflict: the same protocol and port, and the wildcard on either side or the same ip
  std::vector<uint64_t> conflict(K, 0);
  for (uint32_t a = 0; a < K; ++a)
    for (uint32_t b = 0; b < K; ++b) {
      if (t->protocol[a] != t->protocol[b] || t->port[a] != t->port[b]) continue;
      if (a != b && t->ip[a] == t->ip[b]) return bad(BS_E_INVAL, "an entry is listed twice");
      if (t->ip[a] == BS_HOSTPORT_IP_ANY || t->ip[b] == BS_HOSTPORT_IP_ANY || t->ip[a] == t->ip[b])
        conflict[a] |= 1ull << b;
    }
  uint64_t any = 0;
  for (uint32_t n = 0; n < N; ++n) any |= t->used[n];
  if (K < 64 && (any >> K)) return bad(BS_E_INDEX, "a used bit is >= n_entries");
  BS_DEVICE_GUARD(e);
  if (int rc = upload_vec(e, e->hp.d_used, t->used, N, e->Npad)) return rc;
  CK(cudaStreamSynchronize(e->s));
  e->hp.h_conflict = std::move(conflict);
  e->hp.h_used.assign(t->used, t->used + N);
  e->hp.h_conflict.resize(BS_HOSTPORT_MAX, 0);   // want bits past n_entries are refused at evaluation
  e->hp.entries = K;
  e->hp.have_node = true;
  e->hp.dirty = true;
  if (e->hp.on) e->filt.assign_dirty = e->classes_dirty = e->pod_classes_dirty = true;   // new conflict masks
  e->evaluated = false;
  return BS_OK;
}

int bs_upload_pod_host_ports(bs_engine* e, uint32_t n_pods, const uint64_t* want) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  const Refuse bad{e, "bs_upload_pod_host_ports"};
  e->hp.have_pod = false;
  if (int rc = bad.shape(POD_SIDE, n_pods)) return rc;
  if (n_pods && !want) return bad(BS_E_INVAL, "null want");
  e->hp.h_want.assign(want, want + n_pods);
  uint64_t all = 0;
  for (uint32_t p = 0; p < n_pods; ++p) all |= want[p];
  e->hp.want_all = all;
  e->hp.have_pod = true;
  e->filt.assign_dirty = e->classes_dirty = e->pod_classes_dirty = true;   // the pods' fit classes carry the mask
  e->evaluated = false;
  return BS_OK;
}

int bs_upload_bound_host_ports(bs_engine* e, uint32_t n_pods, const uint64_t* ports) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  const Refuse bad{e, "bs_upload_bound_host_ports"};
  e->hp.have_bound = false;
  if (!e->have_bound) return bad(BS_E_STATE, "upload the bound-pod table first");
  if (n_pods != e->V) return bad(BS_E_INVAL, "n_pods differs from the bound-pod table's");
  if (n_pods && !ports) return bad(BS_E_INVAL, "null ports");
  // the bits are checked against the node side when a preemption starts: the sides may come in any order
  const uint32_t V = e->V, N = e->N, Vp = std::max(V, 1u);
  BS_DEVICE_GUARD(e);
  if (int rc = upload_vec(e, e->hp.d_bstage, ports, V, Vp)) return rc;   // table order
  CK(e->hp.d_bports.ensure((size_t)Vp * 8));
  CK(e->hp.d_bsuf.ensure((size_t)Vp * 8));
  if (N) {
    preempt_ports_prep_kernel<<<cdiv(N, 256), 256, 0, e->s>>>(e->d_brow.as<uint32_t>(), e->d_bidx.as<uint32_t>(),
                                                             e->hp.d_bstage.as<uint64_t>(), e->hp.d_bports.as<uint64_t>(),
                                                             e->hp.d_bsuf.as<uint64_t>(), N);
    ++e->launches;
  }
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(e->s));
  e->hp.h_bports.assign(ports, ports + V);
  e->hp.have_bound = true;
  return BS_OK;
}

int bs_fetch_host_port_reason_rows(bs_engine* e, uint32_t pod0, uint32_t n, uint32_t* counts) {
  if (!e || (n && !counts)) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->evaluated || !(e->out_flags & BS_OUT_REASONS)) return fail(e, BS_E_STATE, "no reason rows materialised");
  if ((uint64_t)pod0 + n > e->P) return BS_E_INDEX;
  if (!n) return BS_OK;
  if (!e->hp.round) {
    memset(counts, 0, (size_t)n * 4);
    return BS_OK;
  }
  BS_DEVICE_GUARD(e);
  CK(cudaMemcpyAsync(counts, e->hp.d_reasons.as<uint32_t>() + pod0, (size_t)n * 4, cudaMemcpyDeviceToHost, e->s));
  CK(cudaStreamSynchronize(e->s));
  return BS_OK;
}

int bs_fetch_priority_rows(bs_engine* e, uint32_t pod0, uint32_t n, int32_t* nodes, int64_t* scores) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->evaluated || !(e->out_flags & BS_OUT_PRIORITY)) return fail(e, BS_E_STATE, "no priority lists materialised");
  if ((uint64_t)pod0 + n > e->P) return BS_E_INDEX;
  BS_DEVICE_GUARD(e);
  const size_t off = (size_t)pod0 * e->topk, cnt = (size_t)n * e->topk;   // device rows are dense [P][K]
  if (cnt && nodes)
    CK(cudaMemcpyAsync(nodes, e->d_prio_node.as<int32_t>() + off, cnt * 4, cudaMemcpyDeviceToHost, e->s));
  if (cnt && scores)
    CK(cudaMemcpyAsync(scores, e->d_prio_score.as<int64_t>() + off, cnt * 8, cudaMemcpyDeviceToHost, e->s));
  CK(cudaStreamSynchronize(e->s));
  return BS_OK;
}

int bs_peer_init(bs_engine* e, uint32_t rank, uint32_t world, uint32_t words_per_rank) {
  if (!e || world == 0 || world > PEER_MAX_WORLD || rank >= world || words_per_rank == 0) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  BS_DEVICE_GUARD(e);
  if (e->peer_attached) return fail(e, BS_E_STATE, "bs_peer_init: detach first");
  const size_t bytes = peer_buf_words(world, words_per_rank) * 4;
  e->d_gather.reset();   // a fresh allocation: the IPC handle names this exact block
  CK(e->d_gather.ensure(bytes));
  CK(e->d_peer_err.ensure(sizeof(int)));
  CK(cudaMemsetAsync(e->d_gather.p, 0, e->d_gather.cap, e->s));
  CK(cudaMemsetAsync(e->d_peer_err.p, 0, sizeof(int), e->s));
  CK(cudaStreamSynchronize(e->s));
  e->peer_rank = rank; e->peer_world = world; e->peer_wpr = words_per_rank; e->peer_seq = 0;
  e->peer_broken = false;
  if (const char* t = getenv("BS_PEER_TIMEOUT_MS")) e->peer_timeout_ns = (unsigned long long)std::max(1, atoi(t)) * 1000000ull;
  return BS_OK;
}

int bs_peer_handle(bs_engine* e, unsigned char handle[64]) {
  if (!e || !handle) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  BS_DEVICE_GUARD(e);
  if (!e->d_gather.p) return fail(e, BS_E_STATE, "bs_peer_handle: bs_peer_init first");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is 64 bytes");
  cudaIpcMemHandle_t h;
  CK(cudaIpcGetMemHandle(&h, e->d_gather.p));
  memcpy(handle, &h, 64);
  return BS_OK;
}

int bs_peer_attach(bs_engine* e, const unsigned char* handles) {
  if (!e || !handles) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  BS_DEVICE_GUARD(e);
  if (!e->d_gather.p) return fail(e, BS_E_STATE, "bs_peer_attach: bs_peer_init first");
  if (e->peer_attached) return fail(e, BS_E_STATE, "bs_peer_attach: already attached");
  for (uint32_t r = 0; r < e->peer_world; ++r) {
    if (r == e->peer_rank) { e->peer_ptr[r] = e->d_gather.p; continue; }
    cudaIpcMemHandle_t h;
    memcpy(&h, handles + (size_t)r * 64, 64);
    void* p = nullptr;
    cudaError_t er = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
    if (er != cudaSuccess) {
      for (uint32_t q = 0; q < r; ++q)
        if (q != e->peer_rank && e->peer_ptr[q]) { cudaIpcCloseMemHandle(e->peer_ptr[q]); e->peer_ptr[q] = nullptr; }
      e->err = std::string("cudaIpcOpenMemHandle: ") + cudaGetErrorString(er);
      cudaGetLastError();
      return BS_E_CUDA;
    }
    e->peer_ptr[r] = p;
  }
  e->peer_attached = true;
  return BS_OK;
}

int bs_peer_detach(bs_engine* e) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  BS_DEVICE_GUARD(e);
  if (e->s) cudaStreamSynchronize(e->s);
  if (e->s4) cudaStreamSynchronize(e->s4);
  for (uint32_t r = 0; r < e->peer_world; ++r) {
    if (r != e->peer_rank && e->peer_ptr[r]) cudaIpcCloseMemHandle(e->peer_ptr[r]);
    e->peer_ptr[r] = nullptr;
  }
  e->peer_attached = false;
  e->peer_broken = false;
  e->peer_seq = 0;
  // A new epoch may attach this buffer again without bs_peer_init: its round 1 must not find the last epoch's words
  // and round numbers in the flags.  The peers' pushes of the last round have landed (this rank's wait for it
  // finished above), and no peer pushes the next epoch before every rank has attached again.
  if (e->d_gather.p && e->s) {
    CK(cudaMemsetAsync(e->d_gather.p, 0, e->d_gather.cap, e->s));
    CK(cudaMemsetAsync(e->d_peer_err.p, 0, sizeof(int), e->s));
    CK(cudaStreamSynchronize(e->s));
  }
  return BS_OK;
}

int bs_peer_join(bs_engine* e) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  BS_DEVICE_GUARD(e);
  if (e->peer_attached && e->peer_seq) CK(cudaStreamWaitEvent(e->s, e->ev_gath, 0));
  return BS_OK;
}

int bs_fetch_gathered_admit(bs_engine* e, uint32_t* words) {
  if (!e || !words) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->peer_attached || !e->peer_seq) return fail(e, BS_E_STATE, "bs_fetch_gathered_admit: no exchanged round");
  BS_DEVICE_GUARD(e);
  int rc = peer_check_locked(e);   // waits for the round's slots to land (stream s4)
  if (rc) return rc;
  const size_t n = (size_t)e->peer_world * e->peer_wpr;
  CK(cudaMemcpyAsync(words, e->d_gather.as<uint32_t>() + (size_t)(e->peer_seq & 1u) * n, n * 4, cudaMemcpyDeviceToHost, e->s4));
  CK(cudaStreamSynchronize(e->s4));
  return BS_OK;
}

int bs_set_profiling(bs_engine* e, int on) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  e->profiling = on != 0;
  return BS_OK;
}

int bs_kernel_ms(bs_engine* e, int k, float* ms, uint32_t* launches) {
  if (!e || k < 0 || k >= BS_K_COUNT) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  if (launches) *launches = e->k_launches[k];
  if (ms) {
    *ms = 0.f;
    if (e->profiling && e->k_valid[k]) {
      BS_DEVICE_GUARD(e);
      CK(cudaEventSynchronize(e->ev_b[k]));
      CK(cudaEventElapsedTime(ms, e->ev_a[k], e->ev_b[k]));
    }
  }
  return BS_OK;
}

uint64_t bs_launch_count(const bs_engine* e) { return e ? e->launches : 0; }

int bs_fit_shape(bs_engine* e, uint32_t* wide, uint32_t* narrow, uint32_t* scaled) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->lane_map_valid) return fail(e, BS_E_STATE, "bs_fit_shape: evaluate first");
  if (wide) *wide = e->lane_map.LW;
  if (narrow) *narrow = e->lane_map.LN;
  if (scaled) *scaled = e->lane_map.LS;
  return BS_OK;
}

int bs_score_memory(bs_engine* e, uint32_t* supported, uint32_t* compressed) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->d_score.p) return fail(e, BS_E_STATE, "bs_score_memory: no score matrix (evaluate with BS_OUT_SCORE first)");
  if (supported) *supported = (uint32_t)e->d_score.a.supported;
  if (compressed) *compressed = e->d_score.a.compressed() ? 1u : 0u;
  return BS_OK;
}

int bs_fit_lanes(bs_engine* e, uint8_t* kind, uint8_t* unit) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->lane_map_valid) return fail(e, BS_E_STATE, "bs_fit_lanes: evaluate first");
  const LaneMap& lm = e->lane_map;
  uint8_t k[BS_MAX_LANES] = {}, u[BS_MAX_LANES] = {};
  for (uint32_t s = 0; s < lm.LN; ++s) k[lm.narrow[s]] = 1;
  for (uint32_t s = 0; s < lm.LS; ++s) {
    k[lm.scaled[s]] = 2;
    u[lm.scaled[s]] = lm.sunit[s];
  }
  for (uint32_t d = 0; d < e->L; ++d) {
    if (kind) kind[d] = k[d];
    if (unit) unit[d] = u[d];
  }
  return BS_OK;
}

int bs_sort_shape(bs_engine* e, uint32_t* kernel, uint32_t* grid, uint32_t* group_passes, uint32_t* pod_passes) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  if (!e->sort_shape.valid) return fail(e, BS_E_STATE, "bs_sort_shape: evaluate first");
  if (kernel) *kernel = e->sort_shape.kernel;
  if (grid) *grid = e->sort_shape.grid;
  if (group_passes) *group_passes = e->sort_shape.group_passes;
  if (pod_passes) *pod_passes = e->sort_shape.pod_passes;
  return BS_OK;
}

int bs_replay_shape(bs_engine* e, uint32_t* cached, uint32_t* fitmask, uint32_t* n_rep, uint32_t* n_blocks,
                    uint32_t* bucket_size, uint32_t* n_buckets, uint32_t* lo, uint32_t* monotone) {
  if (!e) return BS_E_INVAL;
  std::lock_guard<std::mutex> lk(e->mu);
  const auto& r = e->replay_shape;
  if (!r.valid) return fail(e, BS_E_STATE, "bs_replay_shape: walk first");
  if (cached) *cached = r.cached;
  if (fitmask) *fitmask = r.fitmask;
  if (n_rep) *n_rep = r.n_rep;
  if (n_blocks) *n_blocks = r.n_blocks;
  if (bucket_size) *bucket_size = r.bucket_size;
  if (n_buckets) *n_buckets = r.n_buckets;
  if (lo) *lo = r.lo;
  if (monotone) *monotone = r.monotone;
  return BS_OK;
}

}  // extern "C"
