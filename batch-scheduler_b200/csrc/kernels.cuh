// kernels.cuh — sm_90a kernels of the gang-scheduling feasibility engine.
//
// Every kernel cites the reference lines it restates (tenstack/batch-scheduler,
// pkg/scheduler/core/core.go).  All arithmetic is int64 / uint32 / one float32
// multiply per node lane; there is no dense contraction, so no tensor cores.
// Tables are lane-major SoA in HBM (see include/bsched.h); the node table is
// padded to a multiple of NODE_TILE so tiles can be moved with 1-D TMA bulk
// copies (cp.async.bulk, 16-byte granules).
#pragma once
#include <type_traits>

#include "common.cuh"

namespace bsk {

// round-global scalars living in device memory (no host sync inside a round)
struct RoundState {
  int32_t max_group;      // findMaxPG winner or -1
  uint32_t max_finished;
  uint32_t max_matched;   // matched[max_group]
  int32_t case_a;         // 1: matched==0 branch (core.go:136), pct 1.0, need of the pod's own group
  int32_t ref_panic;      // findMaxPG would divide by zero
  int32_t max_class;      // rep class of max_group (case B)
  int32_t no_nodes;       // empty snapshot list: every cluster check is false (core.go:604,631)
  int32_t pad1;
  int64_t base_need[BS_MAX_LANES]; // getPreAllocatedResource(max, matched) (case B, core.go:157)
  uint32_t base_present;
};

// per rep-class statistics of the ordered prefix scan (compareClusterResourceAndRequire)
struct ClassStats {
  int64_t maxv[BS_MAX_LANES];    // max prefix value per lane over visited prefixes (present ones for scalars)
  int32_t argmax[BS_MAX_LANES];  // a prefix index attaining it (-1 none)
  uint32_t any_absent;           // scalar lanes absent at some visited prefix
  int32_t last_visited;          // last visited node index, -1 if none
};

// ---------------------------------------------------------------------------
__device__ __forceinline__ int64_t scale_f32(int64_t alloc, float pct) {
  // core.go:656-659,667: int64(float32(alloc) * percent) — RN convert, RN multiply
  // (no FMA contraction possible on a lone multiply), truncating convert back.
  return __float2ll_rz(__fmul_rn(__ll2float_rn(alloc), pct));
}

__device__ __forceinline__ bool node_skipped(uint8_t f) {
  // core.go:606-617
  return (f & (BS_NODE_NIL | BS_NODE_NO_NODE | BS_NODE_UNSCHEDULABLE)) != 0;
}

__device__ __forceinline__ bool check_fit(uint64_t label, uint64_t taint, uint64_t sel, uint64_t tol) {
  // core.go:741-759 with both predicates pre-encoded as bit sets
  return ((label & sel) == sel) && ((taint & ~tol) == 0);
}

struct NodeTab {
  const int64_t* alloc;      // [L][Npad]
  const int64_t* requested;  // [L][Npad]
  const int32_t* pod_count;
  const uint32_t* alloc_present;
  const uint32_t* req_present;
  const uint64_t* label;
  const uint64_t* taint;
  const uint8_t* flags;
  const uint32_t* aff_bits;  // [n_aff][aff_W] host-evaluated node predicates (bs_upload_affinity), or null
  uint32_t N, Npad, L, aff_W;
};

// The part of PodMatchNodeSelector the 64-bit masks cannot carry (required nodeAffinity terms: In / NotIn /
// Exists / DoesNotExist / Gt / Lt, ORed terms; core.go:741-759 -> predicates.PodMatchNodeSelector): the
// caller evaluates each distinct affinity class against every node and uploads one bit per (class, node).
__device__ __forceinline__ bool aff_ok(const NodeTab& t, uint32_t aff, uint32_t i) {
  return aff == BS_AFF_NONE || ((t.aff_bits[(size_t)aff * t.aff_W + (i >> 5)] >> (i & 31)) & 1u);
}

// singleNodeResource (core.go:634-670) for node i and class (sel,tol,aff) at pct;
// returns the scalar presence mask; v[] gets every lane (zeros when unfit).
template <int MAXL>
__device__ __forceinline__ uint32_t single_node_resource(const NodeTab& t, uint32_t i, uint64_t sel,
                                                         uint64_t tol, uint32_t aff, float pct, int64_t* v) {
#pragma unroll
  for (int d = 0; d < MAXL; ++d) v[d] = 0;
  const uint8_t f = t.flags[i];
  if (f & BS_NODE_TAINTS_ERR) return 0;                                  // :639-641
  if (!check_fit(t.label[i], t.taint[i], sel, tol) || !aff_ok(t, aff, i)) return 0;   // :642-645
  int64_t pc = t.requested[(size_t)LANE_PODS * t.Npad + i];              // :650-653
  if (pc == 0) pc = t.pod_count[i];
  v[LANE_PODS] = scale_f32(t.alloc[(size_t)LANE_PODS * t.Npad + i], pct) - pc;  // :656
#pragma unroll
  for (int d = 0; d < 3; ++d)                                            // :657-659
    v[d] = scale_f32(t.alloc[(size_t)d * t.Npad + i], pct) - t.requested[(size_t)d * t.Npad + i];
  const uint32_t both = t.alloc_present[i] & t.req_present[i] & ~0xFu;   // :662-666
  uint32_t present = 0;
#pragma unroll
  for (int d = 4; d < MAXL; ++d) {
    if (d < (int)t.L && (both >> d) & 1u) {
      v[d] = scale_f32(t.alloc[(size_t)d * t.Npad + i], pct) - t.requested[(size_t)d * t.Npad + i]; // :667
      present |= 1u << d;
    }
  }
  return present;
}

// compareResourceAndRequire (core.go:672-699) on lane arrays + presence masks
__device__ __forceinline__ bool compare_res(const int64_t* left, uint32_t lpres, const int64_t* req,
                                            uint32_t rpres, int L) {
  bool ok = (left[LANE_MEM] >= req[LANE_MEM]) & (left[LANE_CPU] >= req[LANE_CPU]) &
            (left[LANE_EPH] >= req[LANE_EPH]) & (left[LANE_PODS] >= req[LANE_PODS]);
  for (int d = 4; d < L; ++d) {
    const uint32_t bit = 1u << d;
    if (!(rpres & bit)) continue;                 // :686 only keys of req
    if (!(lpres & bit)) ok &= (req[d] == 0);      // :688-692
    else ok &= (req[d] <= left[d]);               // :694
  }
  return ok;
}

// One lane of compareResourceAndRequire (core.go:672-699) against node_left_kernel's full-width residuals (left_full,
// left_present | 0xF): short when the key is present and left < req (:694), or absent and req != 0 (:688-692).  The
// caller applies it to lanes 0-3 and to the scalar lanes the pod requests.  Reason rows count the short lanes; the
// priority lists take a node as fitting when its gate bit is set and no lane is short.
__device__ __forceinline__ bool lane_short(bool present, int64_t left, int64_t req) {
  return present ? left < req : req != 0;
}

// ---------------------------------------------------------------------------
// The resource priorities (include/bsched.h, DESIGN.md §2 "Resource priorities"): kube-scheduler v1.17's
// NodeResourcesLeastAllocated, NodeResourcesMostAllocated and NodeResourcesBalancedAllocation for one (pod, node)
// pair.  Shared by the round's priority lists (priority.cuh) and bs_replay_priority's node choice (replay.cuh).

// floor(100 r / c) for 0 <= r <= c, 0 < c <= 2^56 (the node table's bound), and whether the division is exact.  The
// quotient lies in [0, 100]; a float32 estimate (both operands rounded to nearest, then __fdividef: relative error below 2^-21 in all) is within
// 100 * 2^-21 of it, so its truncation is the quotient or one off, and one exact int64 remainder test corrects it.
// No 64-bit division subroutine runs.
__device__ __forceinline__ int64_t pct_quotient(int64_t r, int64_t c, bool& exact) {
  const int64_t num = r * 100;   // <= 100 * 2^56 < 2^63
  int64_t q = (int64_t)__float2int_rz(__fdividef(__ll2float_rn(num), __ll2float_rn(c)));
  int64_t rem = num - q * c;
  if (rem < 0) { --q; rem += c; }
  else if (rem >= c) { ++q; rem -= c; }
  exact = rem == 0;
  return q;
}

// fractionOfCapacity [upstream, from memory]: capacity 0 counts as full; else IEEE binary64 r / c, round to nearest
__device__ __forceinline__ double cap_fraction(int64_t r, int64_t c) {
  return c == 0 ? 1.0 : __ddiv_rn(__ll2double_rn(r), __ll2double_rn(c));
}

struct ScoreWeights {
  uint32_t least, most, balanced;
};

// The weighted score of one (pod, node) pair, r = non-zero requests with the pod added, c = allocatable (unscaled):
//   least(r, c) = (c - r) * 100 / c = 100 - ceil(100 r / c),  most(r, c) = floor(100 r / c)   (0 when c == 0 or r > c)
//   Balanced = (1 - |fc - fm|) * 100 truncated toward zero (0 when a fraction is >= 1); __double2ll_rz saturates, so a
//   product below -2^63 (a negative allocatable) gives INT64_MIN
// and the sum w_least * Least + w_most * Most + w_balanced * Balanced wraps in two's complement.
__device__ __forceinline__ int64_t pair_score(int64_t r_cpu, int64_t c_cpu, int64_t r_mem, int64_t c_mem, ScoreWeights w) {
  uint64_t s = 0;
  if (w.least | w.most) {
    int64_t least = 0, most = 0;
    if (c_cpu != 0 && r_cpu <= c_cpu) {
      bool ex;
      const int64_t q = pct_quotient(r_cpu, c_cpu, ex);
      most += q;
      least += 100 - q - (ex ? 0 : 1);
    }
    if (c_mem != 0 && r_mem <= c_mem) {
      bool ex;
      const int64_t q = pct_quotient(r_mem, c_mem, ex);
      most += q;
      least += 100 - q - (ex ? 0 : 1);
    }
    s += (uint64_t)w.least * (uint64_t)(least / 2) + (uint64_t)w.most * (uint64_t)(most / 2);
  }
  if (w.balanced) {
    const double fc = cap_fraction(r_cpu, c_cpu), fm = cap_fraction(r_mem, c_mem);
    int64_t b = 0;
    if (!(fc >= 1.0 || fm >= 1.0)) b = __double2ll_rz(__dmul_rn(__dsub_rn(1.0, fabs(__dsub_rn(fc, fm))), 100.0));
    s += (uint64_t)w.balanced * (uint64_t)b;
  }
  return (int64_t)s;
}

// kube-scheduler v1.17's RequestedToCapacityRatio priority (include/bsched.h bs_set_ratio_priority, DESIGN.md §2).
// The shape is expanded once on the host into table[u] = shape(u), u = 0..100; the kernels copy it to shared memory
// (the index varies per thread: constant memory would serialize the reads).
constexpr int RATIO_TABLE = 101;
struct RatioSetting {
  const int32_t* table;             // [RATIO_TABLE] in device memory
  uint32_t lane_w[BS_MAX_LANES];    // weight per lane, 0 = not scored (lane 3 and lanes >= L are always 0)
  uint32_t mask;                    // lanes with a non-zero weight
  uint32_t weight;                  // the priority's weight in the total
  uint32_t num0, den0;              // the resources with capacity 0 everywhere: shape(100) * absent_weight and
                                    // absent_weight, or 0 and 0 when shape(100) == 0
};

// One resource's score shape(util) [upstream, from memory]:
//   util = c == 0 || r > c ? 100 : 100 - (c - r) * 100 / c     (int64, wrapping, division truncating toward zero)
// For 0 <= r <= c (so 0 < c <= 2^56) that is ceil(100 r / c) = q + (exact ? 0 : 1) with pct_quotient's q.  Any
// other pair (r < 0, which also covers c < 0) takes the exact path in Go's wrapping arithmetic; it is rare.
// The clamp to [0, 100] before the lookup is exact: util < 0 lies below the first point, whose utilization is >= 0,
// so shape gives s_0 = shape(0); util > 100 lies above the last point, so shape gives the last score = shape(100).
__device__ __forceinline__ int32_t ratio_lane_score(const int32_t* tab, int64_t r, int64_t c) {
  int64_t util = 100;
  if (c != 0 && r <= c) {
    if (r >= 0) {
      bool ex;
      const int64_t q = pct_quotient(r, c, ex);
      util = q + (ex ? 0 : 1);
    } else {
      const int64_t prod = (int64_t)(((uint64_t)c - (uint64_t)r) * 100u);
      const int64_t q = c == -1 ? (int64_t)(0 - (uint64_t)prod) : prod / c;   // Go: x / -1 wraps, never traps
      util = (int64_t)(100u - (uint64_t)q);
    }
  }
  return tab[util < 0 ? 0 : util > 100 ? 100 : util];
}

// Adds one weighted resource to the average: a resource that scores 0 drops out (upstream's resourceScore > 0).
__device__ __forceinline__ void ratio_accumulate(int32_t s, uint32_t w, uint32_t& num, uint32_t& den) {
  if (s > 0) { num += (uint32_t)s * w; den += w; }
}

// Ratio = math.Round(float64(num) / float64(den)), 0 when den == 0.  With den <= 2^24 and num <= 100 den, this is
// floor((2 num + den) / (2 den)): num and den are exact in binary64, and the rounded quotient is within 100 * 2^-53
// of num / den, while a quotient that is not a half-integer lies at least 1 / (2 den) >= 2^-25 from one; so the
// binary64 quotient sits on the same side of every half-integer as the exact one, and an exact half-integer rounds
// away from zero in both.  The division: a float32 estimate (relative error below 2^-21, quotient <= 100.5) is the
// quotient or one off, and one exact remainder test corrects it, as in pct_quotient.
__device__ __forceinline__ int64_t ratio_round(uint32_t num, uint32_t den) {
  if (!den) return 0;
  const int64_t x = 2 * (int64_t)num + den, y = 2 * (int64_t)den;
  int64_t q = (int64_t)__float2int_rz(__fdividef(__ll2float_rn(x), __ll2float_rn(y)));
  const int64_t rem = x - q * y;
  if (rem < 0) --q;
  else if (rem >= y) ++q;
  return q;
}

// weight * Ratio as the unsigned addend of a score (the total wraps in two's complement)
__device__ __forceinline__ uint64_t ratio_term(uint32_t weight, uint32_t num, uint32_t den) {
  return (uint64_t)weight * (uint64_t)ratio_round(num, den);
}

// The round's kernels.  A translation unit that needs only the helpers (priority_inst.cu, replay_inst.cu) defines
// BS_KERNELS_HELPERS_ONLY, so that these external kernels are defined once, in engine.cu; the group and findMaxPG
// helpers the walk shares sit between guarded stretches.
#ifndef BS_KERNELS_HELPERS_ONLY
// node_left_kernel's per-node code, shared with bs_preempt_walk's commit step: the scalar keys of the residuals
// (alloc_present & req_present) and lane d's residual at percent 1.0 (singleNodeResource core.go:647-668), or
// present = false when d is a scalar lane without the key.
__device__ __forceinline__ uint32_t node_left_keys(const NodeTab& t, uint32_t i) {
  return t.alloc_present[i] & t.req_present[i] & ~0xFu;
}
__device__ __forceinline__ int64_t node_lane_left(const NodeTab& t, uint32_t i, uint32_t both, uint32_t d,
                                                  bool& present) {
  present = true;
  if (d == LANE_PODS) {
    int64_t pc = t.requested[(size_t)LANE_PODS * t.Npad + i];
    if (pc == 0) pc = t.pod_count[i];
    return scale_f32(t.alloc[(size_t)LANE_PODS * t.Npad + i], 1.0f) - pc;
  }
  if (d >= 4 && !((both >> d) & 1u)) { present = false; return 0; }
  return scale_f32(t.alloc[(size_t)d * t.Npad + i], 1.0f) - t.requested[(size_t)d * t.Npad + i];
}

// ---------------------------------------------------------------------------
// K1  node_left_kernel — per node: residual capacity at percent 1.0 in the
// sentinel form the fit kernel consumes (absent scalar lane -> ABSENT_LEFT / ABSENT_LEFT32),
// class-independent (checkFit is applied per pod class by class_fit_kernel), split into the
// wide (int64) and narrow (int32) lane tables of the round's LaneMap.
// Restates singleNodeResource core.go:647-668.  Padding nodes (>= N) get zeros.
// left_full (reason rows, BS_OUT_REASONS): every lane in original order as int64, 0 where the key is absent.
__global__ void node_left_kernel(NodeTab t, LaneMap lm, int64_t* __restrict__ left_w /*[LW][Npad]*/,
                                 int32_t* __restrict__ left_n /*[LN+LS][Npad]: narrow lanes, then scaled lanes*/,
                                 uint32_t* __restrict__ left_present /*[Npad]*/,
                                 int64_t* __restrict__ left_plain /*[4][Npad] getLeftResource, or null*/,
                                 int64_t* __restrict__ left_full /*[L][Npad], or null*/) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= t.Npad) return;
  if (left_plain) {
    // getLeftResource (core.go:436-475): plain alloc - requested on the four fixed lanes, no float32
    // factor, no checkFit, never a scalar key (the cloned zero Resource has a nil map, :465-472)
    int64_t v[4] = {0, 0, 0, 0};
    if (i < t.N) {
      int64_t pc = t.requested[(size_t)LANE_PODS * t.Npad + i];
      if (pc == 0) pc = t.pod_count[i];
      for (int d = 0; d < 3; ++d) v[d] = t.alloc[(size_t)d * t.Npad + i] - t.requested[(size_t)d * t.Npad + i];
      v[LANE_PODS] = t.alloc[(size_t)LANE_PODS * t.Npad + i] - pc;
    }
    for (int d = 0; d < 4; ++d) left_plain[(size_t)d * t.Npad + i] = v[d];
  }
  if (i >= t.N) {
    for (uint32_t k = 0; k < lm.LW; ++k) left_w[(size_t)k * t.Npad + i] = 0;
    for (uint32_t k = 0; k < lm.LN + lm.LS; ++k) left_n[(size_t)k * t.Npad + i] = 0;
    if (left_full)
      for (uint32_t d = 0; d < t.L; ++d) left_full[(size_t)d * t.Npad + i] = 0;
    left_present[i] = 0;
    return;
  }
  const uint32_t both = node_left_keys(t, i);
  auto lane_left = [&](uint32_t d, bool& present) -> int64_t { return node_lane_left(t, i, both, d, present); };
  for (uint32_t k = 0; k < lm.LW; ++k) {
    bool pres;
    const int64_t v = lane_left(lm.wide[k], pres);
    left_w[(size_t)k * t.Npad + i] = pres ? v : ABSENT_LEFT;
  }
  for (uint32_t k = 0; k < lm.LN; ++k) {
    bool pres;
    const int64_t v = lane_left(lm.narrow[k], pres);
    left_n[(size_t)k * t.Npad + i] = pres ? (int32_t)v : ABSENT_LEFT32;
  }
  for (uint32_t k = 0; k < lm.LS; ++k) {   // units of 2^sunit: exact, every value of the lane is a multiple
    bool pres;
    const int64_t v = lane_left(lm.scaled[k], pres);
    left_n[(size_t)(lm.LN + k) * t.Npad + i] = pres ? (int32_t)(v >> lm.sunit[k]) : ABSENT_LEFTS;
  }
  if (left_full)
    for (uint32_t d = 0; d < t.L; ++d) {
      bool pres;
      const int64_t v = lane_left(d, pres);
      left_full[(size_t)d * t.Npad + i] = pres ? v : 0;
    }
  left_present[i] = both;
}

// scatter of changed rows into a resident table (bs_update_nodes / bs_update_groups): column c has elem[c]-byte
// elements, [lanes[c]][n] compact in src[c] and [lanes[c]][pitch] in dst[c]; row k goes to row idx[k]
constexpr int SCATTER_MAX_COLS = 8;
struct ScatterCols {
  uint8_t* dst[SCATTER_MAX_COLS];
  const uint8_t* src[SCATTER_MAX_COLS];
  uint32_t elem[SCATTER_MAX_COLS], lanes[SCATTER_MAX_COLS];
  uint32_t n_cols;
};
__global__ void row_scatter_kernel(ScatterCols c, uint32_t pitch, const uint32_t* __restrict__ idx, uint32_t n) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const uint32_t i = idx[k];
  for (uint32_t j = 0; j < c.n_cols; ++j)
    for (uint32_t d = 0; d < c.lanes[j]; ++d) {
      const size_t s = (size_t)d * n + k, t = (size_t)d * pitch + i;
      switch (c.elem[j]) {
        case 1: c.dst[j][t] = c.src[j][s]; break;
        case 4: reinterpret_cast<uint32_t*>(c.dst[j])[t] = reinterpret_cast<const uint32_t*>(c.src[j])[s]; break;
        default: reinterpret_cast<uint64_t*>(c.dst[j])[t] = reinterpret_cast<const uint64_t*>(c.src[j])[s]; break;
      }
    }
}

// generic singleNodeResource table for one class (bs_node_left): left[L][N], present[N]
__global__ void node_left_class_kernel(NodeTab t, uint64_t sel, uint64_t tol, float pct,
                                       int64_t* __restrict__ left, uint32_t* __restrict__ present) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= t.N) return;
  int64_t v[BS_MAX_LANES];
  const uint32_t pres = single_node_resource<BS_MAX_LANES>(t, i, sel, tol, BS_AFF_NONE, pct, v);
  for (uint32_t d = 0; d < t.L; ++d) left[(size_t)d * t.N + i] = v[d];
  present[i] = pres;
}

// K1b  class_fit_kernel — one bit per (pod class, node): node not skipped
// (core.go:606-617), Taints() ok (:639), checkFit (:741-759), and every scalar
// key the class requests with a non-zero amount exists in `left`
// (compareResourceAndRequire :688-690).  Layout is TRANSPOSED for the fit kernel:
// classfit[(c * n_tiles + tile) * 32 + lane] holds, in bit j, the verdict for node
// tile*NODE_TILE + j*32 + lane — exactly the TILE_WORDS nodes lane `lane` owns in
// that tile, so the hot loop needs one coalesced 4-byte load per (pod, tile).  IPF: the MatchInterPodAffinity
// filter is on, and the bit also needs the pass bit of the class's filter class cipf[c] (interpod_filter.cuh; bit
// i % 32 of word ipf_pass[cipf[c] * Wg + i / 32]; BS_IPF_NONE passes).  HP: the PodFitsHostPorts filter is on, and
// the bit also needs (used[i] & cconf[c]) == 0, the node's used host ports against the class's conflict mask.  The
// IPF = HP = false build is the filter-off kernel.
template <bool IPF, bool HP>
__global__ void class_fit_kernel(NodeTab t, const uint32_t* __restrict__ left_present,
                                 const uint64_t* __restrict__ csel, const uint64_t* __restrict__ ctol,
                                 const uint32_t* __restrict__ cnz, const uint32_t* __restrict__ caff,
                                 uint32_t n_classes, uint32_t n_tiles,
                                 ColBits* __restrict__ classfit, uint32_t class0,
                                 const uint32_t* __restrict__ cipf, const uint32_t* __restrict__ ipf_pass, uint32_t Wg,
                                 const uint64_t* __restrict__ cconf, const uint64_t* __restrict__ used) {
  const uint32_t c = class0 + blockIdx.y;   // gridDim.y is capped at 65535: classes go in chunks
  const uint32_t slot = blockIdx.x * blockDim.x + threadIdx.x;  // tile * 32 + lane
  if (slot >= n_tiles * 32 || c >= n_classes) return;
  const uint32_t tile = slot >> 5, lane = slot & 31;
  const uint64_t sel = csel[c], tol = ctol[c];
  const uint32_t nz = cnz[c], aff = caff[c];
  const uint32_t ipf = IPF ? cipf[c] : BS_IPF_NONE;
  const uint64_t conf = HP ? cconf[c] : 0;
  ColBits bits = 0;
#pragma unroll
  for (int j = 0; j < TILE_WORDS; ++j) {
    const uint32_t i = tile * NODE_TILE + j * 32 + lane;
    bool ok = false;
    if (i < t.N) {
      const uint8_t f = t.flags[i];
      ok = !node_skipped(f) && !(f & BS_NODE_TAINTS_ERR) && check_fit(t.label[i], t.taint[i], sel, tol) &&
           aff_ok(t, aff, i) && ((nz & ~left_present[i]) == 0);
      if (IPF && ipf != BS_IPF_NONE) ok = ok && ((ipf_pass[(size_t)ipf * Wg + (i >> 5)] >> (i & 31)) & 1u);
      if (HP && conf) ok = ok && (used[i] & conf) == 0;
    }
    bits |= (ColBits)(ok ? 1u : 0u) << j;
  }
  classfit[(size_t)c * n_tiles * 32 + slot] = bits;
}

// ---------------------------------------------------------------------------
// K1c reason_class_kernel — the class half of a reason row (BS_OUT_REASONS): per fit class, how many nodes are
// unschedulable / unavailable (the guards of core.go:606-617 and :639, in that precedence) and, among the nodes
// past the guards, how many fail the selector (label bits or the affinity-class bit) and the taints (checkFit,
// core.go:741-759; both predicates' reasons count).  Also the class's gate bitmap [c][Wg]: bit n%32 of word n/32
// = node n passes the guards and checkFit, the only nodes whose lanes a reason row inspects.  One thread per node
// (Wg * 32 threads cover the padded table: gate bits of padding nodes are 0), one ballot per warp and bin, one
// global atomic per CTA and bin into class_bins[c][4] (zeroed before the launch).  IPF: the MatchInterPodAffinity
// filter is on, and the kernel also writes gate_ipf = the gate AND the pass bits of the class's filter class, the fit
// set's gate of the priority lists; the gate itself stays the lane sweep's.  HP: the PodFitsHostPorts filter is on;
// the kernel counts into hp_bins[c] (zeroed before the launch) the nodes past the guards whose used host ports
// conflict with the class's conflict mask, whatever their other bins, and gate_ipf also needs no conflict.  The
// IPF = HP = false build is the filter-off kernel.
constexpr int REASON_CLASS_THREADS = 256;
struct HostPortClassArgs {
  const uint64_t* cconf;   // [classes] conflict mask of each fit class
  const uint64_t* used;    // [Npad] used host ports of each node
  uint32_t* hp_bins;       // [classes]
};
template <bool IPF, bool HP>
__global__ void __launch_bounds__(REASON_CLASS_THREADS)
reason_class_kernel(NodeTab t, const uint64_t* __restrict__ csel, const uint64_t* __restrict__ ctol,
                    const uint32_t* __restrict__ caff, uint32_t n_classes, uint32_t Wg,
                    uint32_t* __restrict__ gate, uint32_t* __restrict__ class_bins, uint32_t class0,
                    const uint32_t* __restrict__ cipf, const uint32_t* __restrict__ ipf_pass,
                    uint32_t* __restrict__ gate_ipf, HostPortClassArgs hpa) {
  const uint32_t c = class0 + blockIdx.y;   // gridDim.y is capped at 65535: classes go in chunks
  if (c >= n_classes) return;
  __shared__ uint32_t s_bins[4];
  __shared__ uint32_t s_hp;
  if (threadIdx.x < 4) s_bins[threadIdx.x] = 0;
  if (HP && threadIdx.x == 4) s_hp = 0;
  __syncthreads();
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x, lane = threadIdx.x & 31;
  bool unsched = false, unavail = false, sel_bad = false, taint_bad = false, pass = false, port_bad = false;
  if (i < t.N) {
    const uint8_t f = t.flags[i];
    if (node_skipped(f) || (f & BS_NODE_TAINTS_ERR)) {
      unsched = !(f & (BS_NODE_NIL | BS_NODE_NO_NODE)) && (f & BS_NODE_UNSCHEDULABLE);
      unavail = !unsched;
    } else {
      const uint64_t sel = csel[c], tol = ctol[c];
      const uint64_t label = t.label[i], taint = t.taint[i];
      // check_fit's two predicates one at a time: a neutral taint / label side leaves only the other
      sel_bad = !check_fit(label, 0, sel, 0) || !aff_ok(t, caff[c], i);
      taint_bad = !check_fit(~0ull, taint, 0, tol);
      pass = !sel_bad && !taint_bad;
      if (HP) port_bad = (hpa.used[i] & hpa.cconf[c]) != 0;
    }
  }
  const uint32_t gw = __ballot_sync(0xffffffffu, pass);
  if (lane == 0 && (i >> 5) < Wg) gate[(size_t)c * Wg + (i >> 5)] = gw;
  const uint32_t pw = HP ? __ballot_sync(0xffffffffu, port_bad) : 0u;
  if ((IPF || HP) && lane == 0 && (i >> 5) < Wg) {
    const uint32_t ipf = IPF ? cipf[c] : BS_IPF_NONE;
    const uint32_t g2 = HP ? gw & ~pw : gw;
    gate_ipf[(size_t)c * Wg + (i >> 5)] = ipf == BS_IPF_NONE ? g2 : g2 & ipf_pass[(size_t)ipf * Wg + (i >> 5)];
  }
  if (HP && lane == 0 && pw) atomicAdd(&s_hp, (uint32_t)__popc(pw));
  const uint32_t b0 = __popc(__ballot_sync(0xffffffffu, unsched)), b1 = __popc(__ballot_sync(0xffffffffu, unavail));
  const uint32_t b2 = __popc(__ballot_sync(0xffffffffu, sel_bad)), b3 = __popc(__ballot_sync(0xffffffffu, taint_bad));
  if (lane == 0) {
    if (b0) atomicAdd(&s_bins[0], b0);
    if (b1) atomicAdd(&s_bins[1], b1);
    if (b2) atomicAdd(&s_bins[2], b2);
    if (b3) atomicAdd(&s_bins[3], b3);
  }
  __syncthreads();
  if (threadIdx.x < 4 && s_bins[threadIdx.x]) atomicAdd(&class_bins[(size_t)c * 4 + threadIdx.x], s_bins[threadIdx.x]);
  if (HP && threadIdx.x == 0 && s_hp) atomicAdd(&hpa.hp_bins[c], s_hp);
}

// K1d reason_pod_kernel — the lane bins of a reason row.  A warp takes REASON_PPW pods and sweeps every node 32 at a
// time (lane k owns node base + k); a node counts only when the pod's class gate bit is set.  Lane d is short under
// compareResourceAndRequire's rules (core.go:672-699) with `left` at percent 1.0 from node_left_kernel (left_full,
// left_present): lanes 0-3 when left < req; a scalar lane the pod requests when the node's left lacks the key and
// req != 0, or when req > left.  Every short lane counts (the reference stops at the first).  Counters stay in
// registers, are summed across the warp once at the end, and each (pod, bin) is stored once; bins 0-3 are copied
// from the pod's class.  IPF: the MatchInterPodAffinity filter is on, and a gated node with no short lane that fails
// the filter counts in ipf_rows[p][3] by the step that failed it (E, A, N; interpod_filter.cuh's planes).  HP: the
// PodFitsHostPorts filter is on; hp_rows[p] is copied from the pod's class (reason_class_kernel's hp_bins), and a
// node with a port conflict counts in no ipf_rows bin.  The IPF = HP = false build is the filter-off kernel.
constexpr int REASON_THREADS = 256;
constexpr int REASON_PPW = 4;                                         // pods per warp
constexpr int REASON_PODS_PER_CTA = (REASON_THREADS / 32) * REASON_PPW;
struct ReasonArgs {
  const int64_t* left;          // [L][Npad] left_full
  const uint32_t* left_present; // [Npad]
  const uint32_t* gate;         // [classes][Wg]
  const uint32_t* class_bins;   // [classes][4]
  const int64_t* req;           // [L][P]
  const uint32_t* req_present;  // [P]
  const uint32_t* fit_class;    // [P]
  uint32_t* rows;               // [P][4 + L]
  uint32_t P, N, Npad, Wg, L;
  // IPF only: each fit class's filter class, the planes [3][n_ipf][Wg] (pass, E, A) and the rows [P][3]
  const uint32_t* cipf;
  const uint32_t* ipf_bits;
  uint32_t n_ipf;
  uint32_t* ipf_rows;
};
// HP only: each fit class's conflict mask and port bin, each node's used host ports [Npad] and the rows [P]
struct ReasonHpArgs : ReasonArgs {
  const uint64_t* cconf;
  const uint32_t* hp_bins;
  const uint64_t* used;
  uint32_t* hp_rows;
};
template <bool HP>
using ReasonArgsOf = typename std::conditional<HP, ReasonHpArgs, ReasonArgs>::type;
template <bool IPF, bool HP>
__global__ void __launch_bounds__(REASON_THREADS) reason_pod_kernel(ReasonArgsOf<HP> a) {
  __shared__ int64_t s_req[REASON_THREADS / 32][REASON_PPW][BS_MAX_LANES];
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const uint32_t p0 = (blockIdx.x * (REASON_THREADS / 32) + wid) * REASON_PPW;
  const int L = (int)a.L;
  for (uint32_t k = lane; k < REASON_PPW * BS_MAX_LANES; k += 32) {
    const uint32_t j = k / BS_MAX_LANES, d = k % BS_MAX_LANES, p = p0 + j;
    s_req[wid][j][d] = (p < a.P && d < a.L) ? a.req[(size_t)d * a.P + p] : 0;
  }
  __syncwarp();
  uint32_t rmask[REASON_PPW];   // lanes compared: 0-3 always, scalar lanes the pod requests
  const uint32_t* grow[REASON_PPW];
  const uint32_t* frow[REASON_PPW];   // IPF: the pass plane row of the pod's filter class, or null
  uint64_t conf[REASON_PPW];          // HP: the conflict mask of the pod's class
#pragma unroll
  for (int j = 0; j < REASON_PPW; ++j) {
    const uint32_t p = p0 + j;
    const bool ok = p < a.P;
    rmask[j] = ok ? (a.req_present[p] | 0xFu) : 0u;
    grow[j] = a.gate + (size_t)(ok ? a.fit_class[p] : 0u) * a.Wg;
    if (IPF) {
      const uint32_t f = ok ? a.cipf[a.fit_class[p]] : BS_IPF_NONE;
      frow[j] = f == BS_IPF_NONE ? nullptr : a.ipf_bits + (size_t)f * a.Wg;
    }
    if constexpr (HP) {
      conf[j] = ok ? a.cconf[a.fit_class[p]] : 0ull;
      if (ok && lane == 0) a.hp_rows[p] = a.hp_bins[a.fit_class[p]];
    }
  }
  uint32_t cnt[REASON_PPW][BS_MAX_LANES];
  uint32_t icnt[REASON_PPW][3];
#pragma unroll
  for (int j = 0; j < REASON_PPW; ++j) {
#pragma unroll
    for (int d = 0; d < BS_MAX_LANES; ++d) cnt[j][d] = 0;
#pragma unroll
    for (int k = 0; k < 3; ++k) icnt[j][k] = 0;
  }
  for (uint32_t base = 0; base < a.N; base += 32) {
    const uint32_t i = base + lane, w = base >> 5;
    bool g[REASON_PPW];
    uint32_t any = 0;
#pragma unroll
    for (int j = 0; j < REASON_PPW; ++j) {
      const uint32_t gw = rmask[j] ? grow[j][w] : 0u;   // the word of the padded table: bits >= N are 0
      any |= gw;
      g[j] = (gw >> lane) & 1u;
    }
    if (!any) continue;   // warp-uniform: no pod of the warp looks at these 32 nodes
    const uint32_t lp = a.left_present[i] | 0xFu;   // i < Npad: the padded table is readable
    bool any_short[REASON_PPW];
#pragma unroll
    for (int j = 0; j < REASON_PPW; ++j) any_short[j] = false;
#pragma unroll
    for (int d = 0; d < BS_MAX_LANES; ++d) {
      if (d >= L) break;
      const int64_t v = a.left[(size_t)d * a.Npad + i];
      const bool pres = (lp >> d) & 1u;
#pragma unroll
      for (int j = 0; j < REASON_PPW; ++j) {
        const int64_t r = s_req[wid][j][d];
        const bool shrt = g[j] && ((rmask[j] >> d) & 1u) && lane_short(pres, v, r);
        cnt[j][d] += shrt ? 1u : 0u;
        if (IPF) any_short[j] = any_short[j] || shrt;
      }
    }
    if (IPF) {
      const size_t plane = (size_t)a.n_ipf * a.Wg;
      uint64_t used = 0;
      if constexpr (HP) used = a.used[i];
#pragma unroll
      for (int j = 0; j < REASON_PPW; ++j) {
        if (!g[j] || any_short[j] || !frow[j] || ((frow[j][w] >> lane) & 1u)) continue;
        if (HP && (used & conf[j])) continue;   // GeneralPredicates failed first
        const bool e_bit = (frow[j][plane + w] >> lane) & 1u, a_bit = (frow[j][2 * plane + w] >> lane) & 1u;
        icnt[j][0] += e_bit ? 1u : 0u;
        icnt[j][1] += !e_bit && a_bit ? 1u : 0u;
        icnt[j][2] += !e_bit && !a_bit ? 1u : 0u;
      }
    }
  }
  const uint32_t R = 4 + a.L;
#pragma unroll
  for (int j = 0; j < REASON_PPW; ++j) {
    const uint32_t p = p0 + j;
    uint32_t mine = 0;
#pragma unroll
    for (int d = 0; d < BS_MAX_LANES; ++d) {
      const uint32_t s = __reduce_add_sync(0xffffffffu, cnt[j][d]);
      if (lane == 4 + d) mine = s;
    }
    if (p < a.P) {
      if (lane < 4) mine = a.class_bins[(size_t)a.fit_class[p] * 4 + lane];
      if (lane < R) a.rows[(size_t)p * R + lane] = mine;
    }
    if (IPF) {
      uint32_t im = 0;
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const uint32_t s = __reduce_add_sync(0xffffffffu, icnt[j][k]);
        if (lane == (uint32_t)k) im = s;
      }
      if (p < a.P && lane < 3) a.ipf_rows[(size_t)p * 3 + lane] = im;
    }
  }
}

#endif  // BS_KERNELS_HELPERS_ONLY

// ---------------------------------------------------------------------------
// K2  group preparation: what fillOccupiedObj (core.go:477-512) leaves behind
// once the first pod of each group (table order) has reached it.
struct GroupTab {
  const uint32_t* min_member;
  const uint32_t* scheduled;
  const uint32_t* matched;
  const uint8_t* flags;
  const int64_t* min_res;  // [L][G]
  const uint32_t* min_res_present;
  const uint32_t* rep_class;  // rep-class id of the carried-in pgs.Pod
  uint32_t G, L;
};
struct PodTab {
  const int64_t* req;  // [L][P]
  const uint32_t* req_present;
  const int32_t* gid;
  const uint8_t* flags;
  const uint32_t* fit_class;  // (sel,tol,nzmask) class
  const uint32_t* rep_class;  // (sel,tol) class
  uint32_t P, L;
};
struct GroupEff {
  uint8_t* flags;
  int64_t* min_res;  // [L][G]
  uint32_t* min_res_present;
  uint32_t* rep_class;
  uint32_t* first_pod;  // lowest pod index reaching fillOccupiedObj, 0xffffffff none
  uint32_t* in_round;   // pods of the group in this round
  uint32_t* contrib;    // pods that passed PreFilter and fit somewhere
  uint32_t* done;       // pods whose fit row is finished (ticket)
};

#ifndef BS_KERNELS_HELPERS_ONLY
__global__ void group_reset_kernel(GroupTab g, GroupEff e, uint8_t* __restrict__ new_denied,
                                   uint32_t* __restrict__ admit_bitmap, uint8_t* __restrict__ okA) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < g.G) {
    e.first_pod[i] = 0xffffffffu;
    e.in_round[i] = 0;
    e.contrib[i] = 0;
    e.done[i] = 0;
    new_denied[i] = 0;
    okA[i] = 0;
  }
  if (i < (g.G + 31) / 32) admit_bitmap[i] = 0;
}

__global__ void group_first_pod_kernel(PodTab p, GroupTab g, GroupEff e) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.P) return;
  const int32_t gi = p.gid[i];
  if (gi < 0 || (uint32_t)gi >= g.G) return;
  atomicAdd(&e.in_round[gi], 1u);
  // reaches fillOccupiedObj: not recently permitted (core.go:95-98), group not frozen (:105-110)
  if (p.flags[i] & BS_POD_PERMITTED_RECENTLY) return;
  if (g.flags[gi] & BS_GROUP_DENIED) return;
  atomicMin(&e.first_pod[gi], i);
}

__global__ void group_effective_kernel(PodTab p, GroupTab g, GroupEff e) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= g.G) return;
  uint8_t f = g.flags[i];
  const uint32_t fp = e.first_pod[i];
  uint32_t rc = g.rep_class[i];
  const bool take_pod = fp != 0xffffffffu && !(f & BS_GROUP_HAS_POD);        // core.go:486-488
  const bool take_res = fp != 0xffffffffu && !(f & BS_GROUP_HAS_MINRES);     // core.go:489-493
  if (take_pod) { f |= BS_GROUP_HAS_POD; rc = p.rep_class[fp]; }
  uint32_t mrp = g.min_res_present[i];
  if (take_res) {
    f |= BS_GROUP_HAS_MINRES;
    mrp = p.req_present[fp] & ~0xFu;
    for (uint32_t d = 0; d < g.L; ++d) {
      const bool pres = d < 4 || ((mrp >> d) & 1u);
      e.min_res[(size_t)d * g.G + i] = pres ? p.req[(size_t)d * p.P + fp] : 0;
    }
  } else {
    for (uint32_t d = 0; d < g.L; ++d) e.min_res[(size_t)d * g.G + i] = g.min_res[(size_t)d * g.G + i];
  }
  e.flags[i] = f;
  e.min_res_present[i] = mrp;
  e.rep_class[i] = rc;
}

// getPreAllocatedResource (core.go:774-793) from the effective columns
__device__ __forceinline__ uint32_t pre_allocated(const GroupTab& g, const GroupEff& e, uint32_t gi,
                                                  int64_t matched, int64_t* need) {
  for (uint32_t d = 0; d < BS_MAX_LANES; ++d) need[d] = 0;
  const int64_t mm = (int64_t)g.min_member[gi];
  const int64_t not_finished = matched != 0 ? mm - matched : mm - (int64_t)g.scheduled[gi];  // :778-783
  uint32_t present = 0;
  if (not_finished > 0 && (e.flags[gi] & BS_GROUP_HAS_MINRES)) {                              // :784-788
    present = e.min_res_present[gi];
    for (uint32_t d = 0; d < g.L; ++d) {
      if (d >= 4 && !((present >> d) & 1u)) continue;
      need[d] = (int64_t)((uint64_t)e.min_res[(size_t)d * g.G + gi] * (uint64_t)not_finished);
    }
  }
  if (need[LANE_PODS] == 0) need[LANE_PODS] = mm + 1;                                         // :789-791
  return present;
}

#endif  // BS_KERNELS_HELPERS_ONLY

// K3  findMaxPG (core.go:701-739) as ONE pass with an associative, order-insensitive merge
// that reproduces the sequential table-order scan exactly (tie rule :725-735):
//   F  = max finished over eligible groups;  c0 = lowest index attaining F;
//   Z  = later F-candidates with Status.Scheduled == 0 (the only ones that can take over, :731);
//   winner = c0 unless c0 is "finished" (scheduled >= minMember, :730); then the scan hands over
//   through Z while the holder is finished: the first Z element with minMember != 0 stops it
//   (zgood), otherwise the last Z element holds (zlast).
// Merging two partial states keeps the lower c0; the other side's c0 joins Z if it qualifies.
struct MaxState {
  uint32_t any;      // some eligible group seen
  uint32_t F;        // max finished
  uint32_t c0;       // lowest index with finished == F
  uint32_t c0_flags; // bit0: scheduled >= minMember (holder is finished); bit1: scheduled == 0; bit2: minMember != 0
  uint32_t zgood;    // lowest Z index with minMember != 0, 0xffffffff none
  uint32_t zlast;    // highest Z index + 1, 0 none
  uint32_t panic;
};
__device__ __forceinline__ MaxState max_state_empty() { return MaxState{0u, 0u, 0xffffffffu, 0u, 0xffffffffu, 0u, 0u}; }
__device__ __forceinline__ MaxState max_state_merge(const MaxState& x, const MaxState& y) {
  MaxState r;
  if (!y.any || (x.any && x.F > y.F)) { r = x; r.panic = x.panic | y.panic; return r; }
  if (!x.any || y.F > x.F) { r = y; r.panic = x.panic | y.panic; return r; }
  const MaxState& lo = x.c0 < y.c0 ? x : y;
  const MaxState& hi = x.c0 < y.c0 ? y : x;
  r = lo;
  r.zgood = min(lo.zgood, hi.zgood);
  r.zlast = max(lo.zlast, hi.zlast);
  if (hi.c0_flags & 2u) {            // the displaced c0 has Status.Scheduled == 0: it is a Z element
    if (hi.c0_flags & 4u) r.zgood = min(r.zgood, hi.c0);
    r.zlast = max(r.zlast, hi.c0 + 1);
  }
  r.panic = x.panic | y.panic;
  return r;
}
__device__ __forceinline__ MaxState max_state_shfl_xor(const MaxState& v, int o) {
  MaxState r;
  r.any = __shfl_xor_sync(0xffffffffu, v.any, o);
  r.F = __shfl_xor_sync(0xffffffffu, v.F, o);
  r.c0 = __shfl_xor_sync(0xffffffffu, v.c0, o);
  r.c0_flags = __shfl_xor_sync(0xffffffffu, v.c0_flags, o);
  r.zgood = __shfl_xor_sync(0xffffffffu, v.zgood, o);
  r.zlast = __shfl_xor_sync(0xffffffffu, v.zlast, o);
  r.panic = __shfl_xor_sync(0xffffffffu, v.panic, o);
  return r;
}
__device__ __forceinline__ MaxState max_state_of(const GroupTab& g, const GroupEff& e, uint32_t i) {
  MaxState st = max_state_empty();
  const uint8_t f = e.flags[i];
  if ((f & BS_GROUP_SCHEDULED) || !(f & BS_GROUP_HAS_POD)) return st;   // :706-711
  const uint32_t mm = g.min_member[i], sc = g.scheduled[i];
  uint32_t fin = 0;
  if ((uint32_t)(mm - sc) != 0u) {                                       // :712-714 (uint32: <=0 means ==0)
    if (mm == 0u) st.panic = 1;                                          // :716-717 integer divide by zero
    else fin = (uint32_t)((g.matched[i] + sc) * 1000u) / mm;             // uint32 wrap-around
  }
  st.any = 1; st.F = fin; st.c0 = i;
  st.c0_flags = (sc >= mm ? 1u : 0u) | (sc == 0u ? 2u : 0u) | (mm != 0u ? 4u : 0u);
  return st;
}
__device__ __forceinline__ MaxState max_state_block_reduce(MaxState v, MaxState* s_part /*[32]*/) {
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  for (int o = 16; o; o >>= 1) v = max_state_merge(v, max_state_shfl_xor(v, o));
  if (lane == 0) s_part[wid] = v;
  __syncthreads();
  if (wid == 0) {
    v = lane < nw ? s_part[lane] : max_state_empty();
    for (int o = 16; o; o >>= 1) v = max_state_merge(v, max_state_shfl_xor(v, o));
  }
  return v;  // valid in warp 0
}

#ifndef BS_KERNELS_HELPERS_ONLY
constexpr int FINDMAX_THREADS = 256;
constexpr int FINDMAX_PER_THREAD = 4;
__global__ void __launch_bounds__(FINDMAX_THREADS)
find_max_partial_kernel(GroupTab g, GroupEff e, MaxState* __restrict__ partial) {
  __shared__ MaxState s_part[32];
  MaxState v = max_state_empty();
  const uint32_t base = blockIdx.x * (FINDMAX_THREADS * FINDMAX_PER_THREAD);
#pragma unroll
  for (int k = 0; k < FINDMAX_PER_THREAD; ++k) {
    const uint32_t i = base + k * FINDMAX_THREADS + threadIdx.x;
    if (i < g.G) v = max_state_merge(v, max_state_of(g, e, i));
  }
  v = max_state_block_reduce(v, s_part);
  if (threadIdx.x == 0) partial[blockIdx.x] = v;
}

__global__ void __launch_bounds__(1024)
find_max_final_kernel(GroupTab g, GroupEff e, const MaxState* __restrict__ partial, uint32_t n_partial,
                      RoundState* st, uint32_t n_nodes) {
  __shared__ MaxState s_part[32];
  MaxState v = max_state_empty();
  for (uint32_t i = threadIdx.x; i < n_partial; i += blockDim.x) v = max_state_merge(v, partial[i]);
  v = max_state_block_reduce(v, s_part);
  if (threadIdx.x == 0) {
    const bool none = !v.any;
    uint32_t winner = v.c0;
    if (!none && (v.c0_flags & 1u)) {
      if (v.zgood != 0xffffffffu) winner = v.zgood;
      else if (v.zlast != 0) winner = v.zlast - 1;
    }
    st->ref_panic = (int32_t)v.panic;
    st->no_nodes = n_nodes == 0 ? 1 : 0;
    st->max_group = none ? -1 : (int32_t)winner;
    st->max_finished = none ? 0u : v.F;
    st->max_matched = none ? 0u : g.matched[winner];
    st->case_a = (!none && g.matched[winner] == 0) ? 1 : 0;              // core.go:135-136
    st->max_class = none ? -1 : (int32_t)e.rep_class[winner];
    st->base_present = 0;
    for (int d = 0; d < BS_MAX_LANES; ++d) st->base_need[d] = 0;
    if (!none && g.matched[winner] != 0) {
      int64_t need[BS_MAX_LANES];
      st->base_present = pre_allocated(g, e, winner, (int64_t)g.matched[winner], need);  // core.go:157
      for (int d = 0; d < BS_MAX_LANES; ++d) st->base_need[d] = need[d];
    }
  }
}

// ---------------------------------------------------------------------------
// K4  ordered cluster scan — compareClusterResourceAndRequire (core.go:595-632) for a
// representative class: running[i] = sum over visited nodes j<=i of
// singleNodeResource(node_j, class, pct), scalar keys accumulating as a union
// (Resource.Add, :621).  Chunk-parallel: PREFIX_CHUNK nodes per CTA, coalesced loads.
//   prefix_partial_kernel : per (chunk, class) totals of the chunk;
//   prefix_scan_kernel    : offset = sum of the preceding chunks' totals, warp-shuffle scan
//                           inside the chunk, prefixes written, chunk statistics; the last
//                           chunk of a class to finish folds them into ClassStats.
// mode 0: every class c in [c0, c0+gridDim.y) at pct 1.0, only when case A;
// mode 1: the class of the max group at pct 0.7, only when case B (gridDim.y == 1);
// mode 2: unconditional, explicit (sel,tol,pct) — bs_cluster_check.
constexpr int PREFIX_CHUNK = 256;
struct PrefixOut {
  int64_t* pre;       // [classes][L][N]
  uint32_t* present;  // [classes][N]
  ClassStats* stats;  // [classes]
};
struct PrefixScratch {
  int64_t* part;        // [classes][chunks][MAXL] chunk totals
  uint32_t* part_pres;  // [classes][chunks]
  ClassStats* cstats;   // [classes][chunks]
  uint32_t* done;       // [classes] chunks finished (reset by the last one)
};
struct PrefixSel {
  const uint64_t* rsel;
  const uint64_t* rtol;
  const uint32_t* raff;
  uint32_t c0;
  int mode;
  uint64_t xsel, xtol;
  float xpct;
  const RoundState* st;
};
__device__ __forceinline__ bool prefix_select(const PrefixSel& ps, uint32_t slot, uint64_t& sel, uint64_t& tol,
                                              uint32_t& aff, float& pct) {
  if (ps.mode == 0) {
    if (!ps.st->case_a || ps.st->max_group < 0) return false;
    sel = ps.rsel[ps.c0 + slot]; tol = ps.rtol[ps.c0 + slot]; aff = ps.raff[ps.c0 + slot]; pct = 1.0f;
  } else if (ps.mode == 1) {
    if (ps.st->case_a || ps.st->max_group < 0) return false;
    sel = ps.rsel[ps.st->max_class]; tol = ps.rtol[ps.st->max_class]; aff = ps.raff[ps.st->max_class]; pct = 0.7f;
  } else {
    sel = ps.xsel; tol = ps.xtol; aff = BS_AFF_NONE; pct = ps.xpct;
  }
  return true;
}

template <int MAXL>
__global__ void __launch_bounds__(PREFIX_CHUNK)
prefix_partial_kernel(NodeTab t, PrefixSel ps, PrefixScratch sc, uint32_t n_chunks) {
  uint64_t sel, tol;
  uint32_t aff;
  float pct;
  const uint32_t slot = blockIdx.y, chunk = blockIdx.x;
  if (!prefix_select(ps, slot, sel, tol, aff, pct)) return;
  __shared__ int64_t s_tot[PREFIX_CHUNK / 32][MAXL];
  __shared__ uint32_t s_pres[PREFIX_CHUNK / 32];
  const uint32_t i = chunk * PREFIX_CHUNK + threadIdx.x, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int64_t v[MAXL];
#pragma unroll
  for (int d = 0; d < MAXL; ++d) v[d] = 0;
  uint32_t pres = 0;
  if (i < t.N && !node_skipped(t.flags[i])) pres = single_node_resource<MAXL>(t, i, sel, tol, aff, pct, v);
  for (int o = 16; o; o >>= 1) {
#pragma unroll
    for (int d = 0; d < MAXL; ++d) v[d] += __shfl_xor_sync(0xffffffffu, v[d], o);
    pres |= __shfl_xor_sync(0xffffffffu, pres, o);
  }
  if (lane == 0) {
#pragma unroll
    for (int d = 0; d < MAXL; ++d) s_tot[wid][d] = v[d];
    s_pres[wid] = pres;
  }
  __syncthreads();
  if (threadIdx.x < MAXL) {
    int64_t tsum = 0;
    for (int w = 0; w < PREFIX_CHUNK / 32; ++w) tsum += s_tot[w][threadIdx.x];
    sc.part[((size_t)slot * n_chunks + chunk) * MAXL + threadIdx.x] = tsum;
  }
  if (threadIdx.x == 0) {
    uint32_t p = 0;
    for (int w = 0; w < PREFIX_CHUNK / 32; ++w) p |= s_pres[w];
    sc.part_pres[(size_t)slot * n_chunks + chunk] = p;
  }
}

template <int MAXL>
__global__ void __launch_bounds__(PREFIX_CHUNK)
prefix_scan_kernel(NodeTab t, PrefixSel ps, PrefixScratch sc, uint32_t n_chunks, PrefixOut out) {
  uint64_t sel, tol;
  uint32_t aff;
  float pct;
  const uint32_t slot = blockIdx.y, chunk = blockIdx.x;
  if (!prefix_select(ps, slot, sel, tol, aff, pct)) return;
  const uint32_t N = t.N, L = t.L;
  const uint32_t tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  constexpr int NW = PREFIX_CHUNK / 32;
  __shared__ int64_t s_w[NW][MAXL];
  __shared__ uint32_t s_wp[NW];
  __shared__ int64_t s_off[MAXL];
  __shared__ uint32_t s_offp;
  __shared__ int s_amx[NW][MAXL];
  __shared__ int s_last[NW];
  __shared__ uint32_t s_abs[NW];
  __shared__ bool s_is_last;

  // offset of this chunk: totals of every preceding chunk (strided over the CTA, block-reduced)
  int64_t off[MAXL];
#pragma unroll
  for (int d = 0; d < MAXL; ++d) off[d] = 0;
  uint32_t offp = 0;
  for (uint32_t c = tid; c < chunk; c += PREFIX_CHUNK) {
    const int64_t* pp = sc.part + ((size_t)slot * n_chunks + c) * MAXL;
#pragma unroll
    for (int d = 0; d < MAXL; ++d) off[d] += pp[d];
    offp |= sc.part_pres[(size_t)slot * n_chunks + c];
  }
  for (int o = 16; o; o >>= 1) {
#pragma unroll
    for (int d = 0; d < MAXL; ++d) off[d] += __shfl_xor_sync(0xffffffffu, off[d], o);
    offp |= __shfl_xor_sync(0xffffffffu, offp, o);
  }
  if (lane == 0) {
#pragma unroll
    for (int d = 0; d < MAXL; ++d) s_w[wid][d] = off[d];
    s_wp[wid] = offp;
  }
  __syncthreads();
  if (tid < MAXL) {
    int64_t a = 0;
    for (int w = 0; w < NW; ++w) a += s_w[w][tid];
    s_off[tid] = a;
  }
  if (tid == 0) {
    uint32_t p = 0;
    for (int w = 0; w < NW; ++w) p |= s_wp[w];
    s_offp = p;
  }
  __syncthreads();

  // in-chunk inclusive scan
  const uint32_t i = chunk * PREFIX_CHUNK + tid;
  const bool inb = i < N;
  const bool vis = inb && !node_skipped(t.flags[i]);
  int64_t v[MAXL];
#pragma unroll
  for (int d = 0; d < MAXL; ++d) v[d] = 0;
  uint32_t pres = 0;
  if (vis) pres = single_node_resource<MAXL>(t, i, sel, tol, aff, pct, v);
  for (int o = 1; o < 32; o <<= 1) {
#pragma unroll
    for (int d = 0; d < MAXL; ++d) {
      const int64_t w = __shfl_up_sync(0xffffffffu, v[d], o);
      if ((int)lane >= o) v[d] += w;
    }
    const uint32_t wp = __shfl_up_sync(0xffffffffu, pres, o);
    if ((int)lane >= o) pres |= wp;
  }
  __syncthreads();  // s_w reuse
  if (lane == 31) {
#pragma unroll
    for (int d = 0; d < MAXL; ++d) s_w[wid][d] = v[d];
    s_wp[wid] = pres;
  }
  __syncthreads();
#pragma unroll
  for (int d = 0; d < MAXL; ++d) v[d] += s_off[d];
  pres |= s_offp;
  for (uint32_t w = 0; w < wid; ++w) {
#pragma unroll
    for (int d = 0; d < MAXL; ++d) v[d] += s_w[w][d];
    pres |= s_wp[w];
  }
  if (inb) {
    int64_t* pre = out.pre + (size_t)slot * L * N;
#pragma unroll
    for (int d = 0; d < MAXL; ++d)
      if (d < (int)L) pre[(size_t)d * N + i] = v[d];
    out.present[(size_t)slot * N + i] = pres;
  }
  // chunk statistics over visited prefixes
  int64_t mx[MAXL];
  int amx[MAXL];
#pragma unroll
  for (int d = 0; d < MAXL; ++d) {
    const bool has = vis && (d < 4 || ((pres >> d) & 1u));
    mx[d] = has ? v[d] : INT64_MIN;
    amx[d] = has ? (int)i : -1;
  }
  uint32_t absent = vis ? ~pres : 0u;
  int last = vis ? (int)i : -1;
  for (int o = 16; o; o >>= 1) {
#pragma unroll
    for (int d = 0; d < MAXL; ++d) {
      const int64_t om = __shfl_xor_sync(0xffffffffu, mx[d], o);
      const int oa = __shfl_xor_sync(0xffffffffu, amx[d], o);
      if (oa >= 0 && (amx[d] < 0 || om > mx[d] || (om == mx[d] && oa < amx[d]))) { mx[d] = om; amx[d] = oa; }
    }
    absent |= __shfl_xor_sync(0xffffffffu, absent, o);
    last = max(last, __shfl_xor_sync(0xffffffffu, last, o));
  }
  __syncthreads();  // s_w reuse
  if (lane == 0) {
#pragma unroll
    for (int d = 0; d < MAXL; ++d) { s_w[wid][d] = mx[d]; s_amx[wid][d] = amx[d]; }
    s_abs[wid] = absent;
    s_last[wid] = last;
  }
  __syncthreads();
  if (tid == 0) {
    ClassStats cs;
    for (int d = 0; d < BS_MAX_LANES; ++d) { cs.maxv[d] = INT64_MIN; cs.argmax[d] = -1; }
    cs.any_absent = 0;
    cs.last_visited = -1;
    for (int w = 0; w < NW; ++w) {
      for (int d = 0; d < MAXL; ++d)
        if (s_amx[w][d] >= 0 && (cs.argmax[d] < 0 || s_w[w][d] > cs.maxv[d])) {
          cs.maxv[d] = s_w[w][d]; cs.argmax[d] = s_amx[w][d];
        }
      cs.any_absent |= s_abs[w];
      cs.last_visited = max(cs.last_visited, s_last[w]);
    }
    sc.cstats[(size_t)slot * n_chunks + chunk] = cs;
    __threadfence();
    const uint32_t ticket = atomicAdd(&sc.done[slot], 1u);
    s_is_last = (ticket == n_chunks - 1);
  }
  __syncthreads();
  if (s_is_last) {
    // last chunk of this class: fold the chunk statistics (lane d of warp 0 owns lane d)
    __threadfence();
    if (tid < MAXL) {
      int64_t bm = INT64_MIN;
      int ba = -1;
      for (uint32_t c = 0; c < n_chunks; ++c) {
        const ClassStats& cs = sc.cstats[(size_t)slot * n_chunks + c];
        if (cs.argmax[tid] >= 0 && (ba < 0 || cs.maxv[tid] > bm)) { bm = cs.maxv[tid]; ba = cs.argmax[tid]; }
      }
      out.stats[slot].maxv[tid] = bm;
      out.stats[slot].argmax[tid] = ba;
    } else if (tid >= 32 && tid < 32 + BS_MAX_LANES - MAXL) {
      out.stats[slot].maxv[MAXL + tid - 32] = INT64_MIN;
      out.stats[slot].argmax[MAXL + tid - 32] = -1;
    }
    if (tid == 64) {
      uint32_t ab = 0;
      int lv = -1;
      for (uint32_t c = 0; c < n_chunks; ++c) {
        const ClassStats& cs = sc.cstats[(size_t)slot * n_chunks + c];
        ab |= cs.any_absent;
        lv = max(lv, cs.last_visited);
      }
      out.stats[slot].any_absent = ab;
      out.stats[slot].last_visited = lv;
      sc.done[slot] = 0;  // ready for the next launch
    }
  }
}

// Does any visited prefix of class slot `c` satisfy `need`?  Exact:
//   1. per-lane bound: lane d can pass somewhere only if need<=max prefix, or the
//      key is absent somewhere and need==0 (compareResourceAndRequire :686-697);
//   2. candidates: the last visited prefix and each lane's argmax prefix;
//   3. otherwise scan every visited prefix (strided over `nthreads` callers).
// Called by a full warp; returns the warp-uniform answer.
__device__ __forceinline__ bool prefix_satisfies_at(const int64_t* pre, const uint32_t* pp, uint32_t N,
                                                    int L, uint32_t i, const int64_t* need,
                                                    uint32_t npres) {
  int64_t lv[BS_MAX_LANES];
  for (int d = 0; d < L; ++d) lv[d] = pre[(size_t)d * N + i];
  return compare_res(lv, pp[i], need, npres, L);
}

__device__ bool warp_cluster_check(const NodeTab& t, const PrefixOut& po, uint32_t c,
                                   const int64_t* need, uint32_t npres) {
  const uint32_t N = t.N;
  const int L = (int)t.L;
  const ClassStats& cs = po.stats[c];
  const int64_t* pre = po.pre + (size_t)c * L * N;
  const uint32_t* pp = po.present + (size_t)c * N;
  const uint32_t lane = threadIdx.x & 31;
  if (cs.last_visited < 0) return false;  // no node visited: loop body never compares (core.go:631)
  // 1. bounds
  for (int d = 0; d < L; ++d) {
    const bool checked = d < 4 || ((npres >> d) & 1u);
    if (!checked) continue;
    const bool via_present = cs.argmax[d] >= 0 && need[d] <= cs.maxv[d];
    const bool via_absent = d >= 4 && ((cs.any_absent >> d) & 1u) && need[d] == 0;
    if (!via_present && !via_absent) return false;
  }
  // 2. candidates (lane k tests candidate k)
  bool hit = false;
  if ((int)lane <= L) {
    const int idx = lane == 0 ? cs.last_visited : cs.argmax[lane - 1];
    if (idx >= 0) hit = prefix_satisfies_at(pre, pp, N, L, (uint32_t)idx, need, npres);
  }
  if (__any_sync(0xffffffffu, hit)) return true;
  // 3. full ordered scan (any visited prefix)
  for (uint32_t base = 0; base < N; base += 32) {
    const uint32_t i = base + lane;
    bool ok = false;
    if (i < N && !node_skipped(t.flags[i])) ok = prefix_satisfies_at(pre, pp, N, L, i, need, npres);
    if (__any_sync(0xffffffffu, ok)) return true;
  }
  return false;
}

// K5a group_check_kernel — case A (core.go:136-147): per group, need =
// getPreAllocatedResource(own group, 0) against its own rep class at pct 1.0.
// One warp per group; classes [c0, c0+nc) are resident in `po`.
__global__ void group_check_kernel(NodeTab t, GroupTab g, GroupEff e, PrefixOut po, uint32_t c0,
                                   uint32_t nc, const RoundState* __restrict__ st,
                                   uint8_t* __restrict__ okA) {
  if (!st->case_a || st->max_group < 0) return;
  const uint32_t gi = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (gi >= g.G) return;
  if (e.in_round[gi] == 0 || !(e.flags[gi] & BS_GROUP_HAS_POD)) return;
  const uint32_t c = e.rep_class[gi];
  if (c < c0 || c >= c0 + nc) return;
  int64_t need[BS_MAX_LANES];
  const uint32_t npres = pre_allocated(g, e, gi, 0, need);
  const bool ok = warp_cluster_check(t, po, c - c0, need, npres);
  if ((threadIdx.x & 31) == 0) okA[gi] = ok ? 1 : 2;
}

// K5b prefilter_kernel — ScheduleOperation.PreFilter per pod (core.go:88-167) against the
// frozen round state.  Thread per pod.  Case B (core.go:157-165) needs a cluster check per pod
// against the ONE prefix array of the max group's class: the class statistics and the L+1
// candidate prefixes are staged in shared memory once per CTA, so almost every pod is decided
// by <= (L+1)*L compares; a pod the bounds and candidates leave undecided is handed to its warp
// for a cooperative scan over every visited prefix (exactness is never traded).
constexpr int PREFILTER_THREADS = 256;
__global__ void __launch_bounds__(PREFILTER_THREADS)
prefilter_kernel(NodeTab t, PodTab p, GroupTab g, GroupEff e, PrefixOut po,
                 const RoundState* __restrict__ st, const uint8_t* __restrict__ okA,
                 uint8_t* __restrict__ prefilter, uint8_t* __restrict__ new_denied) {
  __shared__ ClassStats s_cs;
  __shared__ int64_t s_cand[BS_MAX_LANES + 1][BS_MAX_LANES];
  __shared__ uint32_t s_cand_pres[BS_MAX_LANES + 1];
  __shared__ int s_cand_idx[BS_MAX_LANES + 1];
  const int L = (int)t.L;
  const uint32_t N = t.N;
  const bool case_b = st->max_group >= 0 && !st->case_a && !st->no_nodes;
  if (case_b) {
    if (threadIdx.x == 0) s_cs = po.stats[0];
    __syncthreads();
    if (threadIdx.x <= (uint32_t)L) {
      const int idx = threadIdx.x == 0 ? s_cs.last_visited : s_cs.argmax[threadIdx.x - 1];
      s_cand_idx[threadIdx.x] = idx;
      if (idx >= 0) {
        for (int d = 0; d < L; ++d) s_cand[threadIdx.x][d] = po.pre[(size_t)d * N + idx];
        s_cand_pres[threadIdx.x] = po.present[idx];
      }
    }
    __syncthreads();
  }
  const uint32_t pi = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t lane = threadIdx.x & 31;
  const bool valid = pi < p.P;
  int32_t gi = BS_GID_NONE;
  uint8_t code = BS_PF_PASS;
  bool deny = false, undecided = false;
  int64_t need[BS_MAX_LANES];
  uint32_t npres = 0;
  if (valid) {
    gi = p.gid[pi];
    const uint8_t pf = p.flags[pi];
    if (gi == BS_GID_NONE) code = BS_PF_PASS;                                   // :89-92
    else if (pf & BS_POD_PERMITTED_RECENTLY) code = BS_PF_PASS;                 // :95-98
    else if (gi < 0 || (uint32_t)gi >= g.G) code = BS_PF_ERR_NOT_FOUND;         // :100-103
    else if (g.flags[gi] & BS_GROUP_DENIED) code = BS_PF_ERR_DENIED;            // :105-110
    else if (pf & BS_POD_OCC_NOREFS) code = BS_PF_ERR_OCCUPIED_NOREFS;          // :504-506
    else if (pf & BS_POD_OCC_MISMATCH) code = BS_PF_ERR_OCCUPIED;               // :507-510
    else if (st->max_group < 0) code = BS_PF_PASS;                              // :127-130
    else if (st->case_a) {                                                      // :136-147
      if (okA[gi] == 2 || st->no_nodes) { code = BS_PF_ERR_NOT_ENOUGH; deny = true; }
    } else if (st->max_group == gi) code = BS_PF_PASS;                          // :150-155
    else {                                                                      // :157-165
      npres = st->base_present;
      const uint32_t rp = p.req_present[pi] & ~0xFu;
      for (int d = 0; d < L; ++d) {                                             // :159 Add(pod require)
        need[d] = st->base_need[d];
        if (d < 4 || ((rp >> d) & 1u)) need[d] += p.req[(size_t)d * p.P + pi];
      }
      npres |= rp;
      // 1. bounds  2. candidates (see warp_cluster_check)  3. cooperative scan if undecided
      bool reject = st->no_nodes || s_cs.last_visited < 0;
      for (int d = 0; d < L && !reject; ++d) {
        const bool checked = d < 4 || ((npres >> d) & 1u);
        if (!checked) continue;
        const bool via_present = s_cs.argmax[d] >= 0 && need[d] <= s_cs.maxv[d];
        const bool via_absent = d >= 4 && ((s_cs.any_absent >> d) & 1u) && need[d] == 0;
        if (!via_present && !via_absent) reject = true;
      }
      if (reject) { code = BS_PF_ERR_NOT_ENOUGH; deny = true; }
      else {
        bool hit = false;
        for (int c = 0; c <= L && !hit; ++c)
          if (s_cand_idx[c] >= 0) hit = compare_res(s_cand[c], s_cand_pres[c], need, npres, L);
        undecided = !hit;
      }
    }
  }
  // cooperative fallback: one undecided pod at a time, the whole warp scans the prefixes
  uint32_t pending = __ballot_sync(0xffffffffu, undecided);
  while (pending) {
    const int src = __ffs(pending) - 1;
    pending &= pending - 1;
    int64_t nd[BS_MAX_LANES];
    for (int d = 0; d < L; ++d) nd[d] = __shfl_sync(0xffffffffu, need[d], src);
    const uint32_t np = __shfl_sync(0xffffffffu, npres, src);
    bool found = false;
    for (uint32_t base = 0; base < N && !found; base += 32) {
      const uint32_t i = base + lane;
      bool ok = false;
      if (i < N && !node_skipped(t.flags[i])) ok = prefix_satisfies_at(po.pre, po.present, N, L, i, nd, np);
      found = __any_sync(0xffffffffu, ok);
    }
    if ((int)lane == src && !found) { code = BS_PF_ERR_NOT_ENOUGH; deny = true; }
  }
  if (valid) {
    prefilter[pi] = code;
    if (deny) new_denied[gi] = 1;                                               // :142,:163
  }
}

// explicit needs against class slot 0 (bs_cluster_check); one warp per need
__global__ void needs_check_kernel(NodeTab t, PrefixOut po, const int64_t* __restrict__ need /*[L][n]*/,
                                   const uint32_t* __restrict__ need_present, uint32_t n_needs,
                                   uint8_t* __restrict__ ok) {
  const uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (i >= n_needs) return;
  int64_t nd[BS_MAX_LANES];
  for (uint32_t d = 0; d < BS_MAX_LANES; ++d) nd[d] = d < t.L ? need[(size_t)d * n_needs + i] : 0;
  const bool r = warp_cluster_check(t, po, 0, nd, need_present[i] & ~0xFu);
  if ((threadIdx.x & 31) == 0) ok[i] = r ? 1 : 0;
}

// groups with no pod in the round are decided up front (core.go:303 on carried-in state)
__global__ void group_idle_admit_kernel(GroupTab g, GroupEff e, uint8_t* __restrict__ admit,
                                        uint32_t* __restrict__ admit_bitmap) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= g.G || e.in_round[i] != 0) return;
  const bool ready = g.matched[i] >= (uint32_t)(g.min_member[i] - g.scheduled[i]);
  admit[i] = ready ? BS_ADMIT : BS_WAIT;
  if (ready) atomicOr(&admit_bitmap[i >> 5], 1u << (i & 31));
}

// K6b  gang_admit_kernel — the per-group half of Permit (core.go:303) as its own launch: one pod per
// thread, runs of equal gid merged inside the warp, one atomic per run, the run that completes the
// group's pod count writes the verdict.  Used when the PreFilter chain runs on a side stream beside
// gang_fit_kernel (its verdicts are needed only here, after both).
struct AdmitArgs {
  const int32_t* gid;
  const uint8_t* prefilter;
  const uint32_t* feasible_count;
  const uint32_t* min_member;
  const uint32_t* scheduled;
  const uint32_t* matched;
  const uint32_t* in_round;
  uint32_t* contrib;
  uint32_t* done;
  uint8_t* admit;
  uint32_t* admit_bitmap;
  uint32_t P, G;
};
__global__ void __launch_bounds__(256) gang_admit_kernel(AdmitArgs a) {
  const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x, lane = threadIdx.x & 31;
  uint32_t my_gid = 0xffffffffu, my_pass = 0;
  if (p < a.P) {
    const int32_t g = a.gid[p];
    if (g >= 0 && (uint32_t)g < a.G) {
      my_gid = (uint32_t)g;
      my_pass = (a.prefilter[p] == BS_PF_PASS && a.feasible_count[p] > 0) ? 1u : 0u;
    }
  }
  const uint32_t prev_gid = __shfl_up_sync(0xffffffffu, my_gid, 1);
  const bool active = my_gid != 0xffffffffu;
  const bool head = active && (lane == 0 || prev_gid != my_gid);
  uint32_t run_pass = my_pass, run_len = active ? 1u : 0u;
#pragma unroll
  for (int o = 1; o < 32; ++o) {
    const uint32_t og = __shfl_down_sync(0xffffffffu, my_gid, o);
    const uint32_t op = __shfl_down_sync(0xffffffffu, my_pass, o);
    // run_len == o  <=>  every lane in between carried the same gid (contiguous run)
    if (head && run_len == (uint32_t)o && lane + o < 32 && og == my_gid) {
      run_pass += op;
      run_len += 1;
    }
  }
  if (head) {
    if (run_pass) atomicAdd(&a.contrib[my_gid], run_pass);
    __threadfence();
    const uint32_t ticket = atomicAdd(&a.done[my_gid], run_len) + run_len;
    if (ticket == a.in_round[my_gid]) {
      // last pod of the group: Permit readiness (core.go:303) on the full count
      __threadfence();
      const uint32_t c = atomicAdd(&a.contrib[my_gid], 0u);
      const uint32_t total = a.matched[my_gid] + c;
      uint8_t verdict;
      if (c == 0) verdict = BS_UNSCHEDULABLE;
      else verdict = (total >= (uint32_t)(a.min_member[my_gid] - a.scheduled[my_gid])) ? BS_ADMIT : BS_WAIT;
      a.admit[my_gid] = verdict;
      if (verdict == BS_ADMIT) atomicOr(&a.admit_bitmap[my_gid >> 5], 1u << (my_gid & 31));
    }
  }
}

// ---------------------------------------------------------------------------
// K7  filter_kernel — ScheduleOperation.Filter / computeResourceSatisfied (core.go:170-191,
// 514-564) for every (pod,node) against the round's max group m (optional, BS_OUT_FILTER):
//   unlabelled -> pass; group missing -> "can not found pod group"; m == own group -> pass (case 1);
//   max group without MinResources -> pass; info == nil -> "SnapShot not initialized";
//   case 2: left >= require(pod) + MinResources(max) -> pass;
//   case 3: !(left >= MinResources(max)) -> pass; else "resource not enough".
// `left` = getLeftResource has NO scalar keys, so a request key passes only with amount 0.
// Warp per FILTER_PPW pods; a lane owns one node of each 32-node step; ballots become bitmap words.
constexpr int FILTER_PPW = 4;
struct FilterArgs {
  const int64_t* left_plain;  // [4][Npad]
  const uint8_t* node_flags;
  const int64_t* req;         // [L][P]
  const uint32_t* req_present;
  const int32_t* gid;
  const int64_t* emin_res;    // [L][G] effective MinResources
  const uint32_t* emin_res_present;
  const uint8_t* eflags;
  const RoundState* st;
  uint32_t* filter_bitmap;    // [Ppad][W]
  uint8_t* filter_code;       // [P]
  uint32_t P, N, Npad, W, G, L;
};
__global__ void __launch_bounds__(256) filter_kernel(FilterArgs a) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t wpod0 = ((blockIdx.x * blockDim.x + threadIdx.x) >> 5) * FILTER_PPW;
  if (wpod0 >= a.P) return;
  const int32_t m = a.st->max_group;
  // MinResources of the max group as a Resource (core.go:525-528)
  int64_t mmr[4] = {0, 0, 0, 0};
  bool has_mr = false, mmr_scalars_zero = true;
  uint32_t mmr_present = 0;
  if (m >= 0 && (a.eflags[m] & BS_GROUP_HAS_MINRES)) {
    has_mr = true;
    mmr_present = a.emin_res_present[m] & ~0xFu;
    for (int d = 0; d < 4; ++d) mmr[d] = a.emin_res[(size_t)d * a.G + m];
    for (uint32_t d = 4; d < a.L; ++d)
      if (((mmr_present >> d) & 1u) && a.emin_res[(size_t)d * a.G + m] != 0) mmr_scalars_zero = false;
  }
  int64_t rq[FILTER_PPW][4];
  uint8_t mode[FILTER_PPW];   // 0 all pass, 1 none pass, 2 general
  bool sc_ok[FILTER_PPW];
#pragma unroll
  for (int r = 0; r < FILTER_PPW; ++r) {
    const uint32_t p = wpod0 + r;
    mode[r] = 1; sc_ok[r] = false;
    for (int d = 0; d < 4; ++d) rq[r][d] = 0;
    if (p >= a.P) continue;
    const int32_t g = a.gid[p];
    uint8_t code = BS_FILTER_PASS;
    if (g == BS_GID_NONE) mode[r] = 0;                                        // core.go:171-174
    else if (g < 0 || (uint32_t)g >= a.G) { mode[r] = 1; code = BS_FILTER_ERR_NOT_FOUND; }  // :177-180
    else if (m < 0) { mode[r] = 1; code = BS_FILTER_REF_PANIC; }              // :525
    else if (m == g || !has_mr) mode[r] = 0;                                  // :531-535, :542-544
    else {
      mode[r] = 2;
      const uint32_t rp = a.req_present[p] & ~0xFu;
      for (int d = 0; d < 4; ++d) rq[r][d] = a.req[(size_t)d * a.P + p] + mmr[d];   // :551-552
      bool ok = true;   // every scalar key of (pod require + MinResources) must sum to 0 (:686-693)
      for (uint32_t d = 4; d < a.L; ++d) {
        const bool in_p = (rp >> d) & 1u, in_m = (mmr_present >> d) & 1u;
        if (!in_p && !in_m) continue;
        const int64_t v = (in_p ? a.req[(size_t)d * a.P + p] : 0) + (in_m ? a.emin_res[(size_t)d * a.G + m] : 0);
        if (v != 0) ok = false;
      }
      sc_ok[r] = ok;
    }
    if (lane == 0) a.filter_code[p] = code;
  }
  uint32_t words[FILTER_PPW];
#pragma unroll
  for (int r = 0; r < FILTER_PPW; ++r) words[r] = 0;
  for (uint32_t base = 0; base < a.Npad; base += 32) {
    const uint32_t n = base + lane;
    int64_t lf[4];
#pragma unroll
    for (int d = 0; d < 4; ++d) lf[d] = a.left_plain[(size_t)d * a.Npad + n];
    const bool in_n = n < a.N;
    const bool nil = in_n && (a.node_flags[n] & BS_NODE_NIL);
    // case 3 (:558): node cannot hold the max group's MinResources
    const bool c3 = !(mmr_scalars_zero && lf[0] >= mmr[0] && lf[1] >= mmr[1] && lf[2] >= mmr[2] && lf[3] >= mmr[3]);
#pragma unroll
    for (int r = 0; r < FILTER_PPW; ++r) {
      bool pass;
      if (mode[r] == 0) pass = in_n;
      else if (mode[r] == 1) pass = false;
      else {
        const bool c2 = sc_ok[r] && lf[0] >= rq[r][0] && lf[1] >= rq[r][1] && lf[2] >= rq[r][2] && lf[3] >= rq[r][3];
        pass = in_n && !nil && (c2 || c3);                                    // :545-563
      }
      const uint32_t bal = __ballot_sync(0xffffffffu, pass);
      if (lane == ((base >> 5) & 31)) words[r] = bal;
    }
    if (((base >> 5) & 31) == 31 || base + 32 >= a.Npad) {
      const uint32_t w = (base >> 5) - ((base >> 5) & 31) + lane;
#pragma unroll
      for (int r = 0; r < FILTER_PPW; ++r) {
        if (w < a.W) a.filter_bitmap[(size_t)(wpod0 + r) * a.W + w] = words[r];
        words[r] = 0;
      }
    }
  }
}

// ---------------------------------------------------------------------------
// K8  peer exchange — all-gather of the admit bitmap over NVLink peer memory (CUDA IPC), as two
// small kernels so that no rank ever spins on its critical path:
//   peer_push_kernel  (main stream, last kernel of round `seq`; one CTA per destination rank):
//       stores this rank's words into slot[seq & 1][rank] of every peer's gather buffer (plain
//       coalesced stores to mapped peer addresses), __threadfence_system(), then publishes
//       flag[seq & 1][rank] = seq at the peer.
//   peer_wait_kernel  (side stream, one warp): waits until flag[seq & 1][r] >= seq for every r,
//       i.e. until every rank's slot of round `seq` has landed here.  Consumers of the gathered
//       bitmap (bs_fetch_gathered_admit, bs_sync, bs_peer_join) order themselves behind it.
// The gather buffer holds TWO slot sets, indexed by the parity of seq.  Slot set seq & 1 last held
// round seq-2; a rank pushes round seq only after its own wait for round seq-1 has finished (the
// engine orders the push behind that event), and a peer publishes its flag for seq-1 only after it
// has consumed round seq-2 (same rule on its side, stream order) — so the overwrite is safe without
// acknowledgements, and the next round's fit kernel runs while the previous round's wait is
// still spinning: a late rank delays its peers only once it is more than one round behind.
// The spin is bounded (globaltimer); on a timeout *err is set, the engine marks the exchange
// broken and every later call fails fast with BS_E_PEER until the ranks detach and re-attach.
constexpr int PEER_MAX_WORLD = 16;
struct PeerArgs {
  uint32_t* peer_buf[PEER_MAX_WORLD];  // mapped base of every rank's gather buffer (own = local)
  const uint32_t* local_bitmap;        // this rank's admit bitmap words
  uint32_t rank, world, words_per_rank, n_words;  // n_words <= words_per_rank valid words
  uint32_t seq;
  int* err;
  unsigned long long timeout_ns;
};
// buffer layout: [2][world][words_per_rank] data | [2][PEER_MAX_WORLD] flags
__host__ __device__ inline size_t peer_buf_words(uint32_t world, uint32_t wpr) {
  return (size_t)2 * world * wpr + 2 * PEER_MAX_WORLD;
}
__device__ __forceinline__ uint32_t* peer_slot(uint32_t* base, uint32_t world, uint32_t wpr, uint32_t parity, uint32_t r) {
  return base + ((size_t)parity * world + r) * wpr;
}
__device__ __forceinline__ uint32_t* peer_flags(uint32_t* base, uint32_t world, uint32_t wpr, uint32_t parity) {
  return base + (size_t)2 * world * wpr + (size_t)parity * PEER_MAX_WORLD;
}
__device__ __forceinline__ unsigned long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__global__ void __launch_bounds__(256) peer_push_kernel(PeerArgs a) {
  const uint32_t r = blockIdx.x, par = a.seq & 1u;
  uint32_t* dst = peer_slot(a.peer_buf[r], a.world, a.words_per_rank, par, a.rank);
  for (uint32_t w = threadIdx.x; w < a.words_per_rank; w += blockDim.x) dst[w] = w < a.n_words ? a.local_bitmap[w] : 0u;
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) {
    volatile uint32_t* f = peer_flags(a.peer_buf[r], a.world, a.words_per_rank, par);
    f[a.rank] = a.seq;
    __threadfence_system();
  }
}
__global__ void __launch_bounds__(32) peer_wait_kernel(PeerArgs a) {
  volatile uint32_t* f = peer_flags(a.peer_buf[a.rank], a.world, a.words_per_rank, a.seq & 1u);
  bool ok = true;
  if (threadIdx.x < a.world) {
    const unsigned long long t0 = global_ns();
    while (f[threadIdx.x] < a.seq) {
      __nanosleep(64);
      if (global_ns() - t0 > a.timeout_ns) { ok = false; break; }
    }
  }
  __threadfence_system();
  if (!ok) *a.err = 1;
}

#endif  // BS_KERNELS_HELPERS_ONLY

}  // namespace bsk
