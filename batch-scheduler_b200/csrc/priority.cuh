// priority.cuh — the resource priorities of a round (BS_OUT_PRIORITY): each pod's K best fitting nodes under
// kube-scheduler v1.17's NodeResourcesLeastAllocated, NodeResourcesMostAllocated and
// NodeResourcesBalancedAllocation (include/bsched.h, DESIGN.md §2 "Resource priorities").
//
// The fit set is the reason rows' (kernels.cuh K1c/K1d): a node fits a pod when its class gate bit is set and no lane
// is short (lane_short over node_left_kernel's full-width residuals), the invariant DESIGN §2 states for reason rows.
// The lists are kept with gang_fit's topk_insert (fit.cuh); the pair scorer pair_score is kernels.cuh's, and with RATIO
// the RequestedToCapacityRatio term (kernels.cuh ratio_*) is added to it; with PREF the TaintToleration and preferred
// NodeAffinity terms (bs_set_node_priority_weights), normalized over the pod's fit set; with LOC the ImageLocality and
// NodePreferAvoidPods terms (bs_set_locality_weights), static per pair, from the pre-pass below; with SPREAD the
// SelectorSpread term (bs_set_spread_weight), normalized over the pod's fit set and its zones; with IPA the
// InterPodAffinity term (bs_set_interpod_weight), from the pre-pass below, normalized over the pod's fit set.
#pragma once
#include "kernels.cuh"
#include "fit.cuh"

#include <type_traits>

namespace bsk {

// K1e priority_pod_kernel — a warp takes PRIO_PPW pods and sweeps every node 32 at a time (lane k owns node
// base + k), as reason_pod_kernel does.  A node fits when the pod's class gate bit is set and no lane it compares is
// short; each fitting pair is scored and offered to the pod's list.  Lists live in shared memory, 32 (score, node)
// entries per pod ordered by score descending, then node ascending; unfilled entries are (INT64_MIN, PRIO_EMPTY) and
// rank after every real entry, including one that scores INT64_MIN.  A fitting pair is a candidate while the list has
// fewer than K fitting nodes, or when it beats the score of entry K-1: nodes come in ascending order, so a later node
// never displaces an equal score.  MAXL bounds the lanes held in registers (5, 9 or 16).  RATIO (chosen by the host
// when the ratio weight is non-zero) adds w_ratio * Ratio to each score; the node's columns of a weighted lane are read
// once per 32-node step and shared by the warp's pods.
constexpr int PRIO_THREADS = 256;
constexpr int PRIO_PPW = 4;                                           // pods per warp
constexpr int PRIO_PODS_PER_CTA = (PRIO_THREADS / 32) * PRIO_PPW;
constexpr int32_t PRIO_EMPTY = 0x7fffffff;                            // node of an unfilled list entry
struct PriorityArgs {
  const int64_t* left;          // [L][Npad] left_full
  const uint32_t* left_present; // [Npad]
  const uint32_t* gate;         // [classes][Wg]
  const int64_t* req;           // [L][P]
  const uint32_t* req_present;  // [P]
  const uint32_t* fit_class;    // [P]
  const int64_t* alloc;         // [L][Npad] the node table's allocatable: rows 0 (cpu) and 1 (memory)
  const int64_t* node_nz;       // [2][Npad] non-zero requests on the node (padding 0)
  const int64_t* pod_nz;        // [2][P]
  int32_t* out_node;            // [P][K]
  int64_t* out_score;           // [P][K]
  ScoreWeights w;
  uint32_t P, N, Npad, Wg, L, K;
};
// RATIO's arguments: also the node table's requested and key masks, and the setting.  A separate type, so that the
// kernel without the ratio term keeps its parameter block (a larger one changed its SASS).
struct PriorityRatioArgs : PriorityArgs {
  const int64_t* node_requested;        // [L][Npad]
  const uint32_t* node_alloc_present;   // [Npad]
  const uint32_t* node_req_present;     // [Npad]
  RatioSetting ratio;
};
// PREF's arguments (bs_upload_node_preferences / bs_upload_pod_preferences): the PreferNoSchedule taints of each node
// and the tolerated ones of each pod, the preferred-affinity class of each pod and the class x node weight table, and
// the two weights.  Derived from the ratio's type for the same reason; the ratio fields are read only with RATIO.
constexpr uint32_t PREF_NONE = 0xffffffffu;   // BS_PREF_NONE
struct PriorityPrefArgs : PriorityRatioArgs {
  const uint64_t* prefer_taints;   // [Npad] (padding 0)
  const int32_t* pref_weights;     // [classes][Npad] (padding 0)
  const uint64_t* prefer_tol;      // [P]
  const uint32_t* pref_class;      // [P] row of pref_weights or PREF_NONE
  uint32_t w_taint, w_naff;
};
// The raw counts of PREF for one (pod, node): t = PreferNoSchedule taints of the node the pod does not tolerate,
// a = the summed weights of the pod's preferred terms the node matches.  A weight of 0 skips its read (uniform).
__device__ __forceinline__ void pref_counts(const PriorityPrefArgs& a, uint64_t taints, uint64_t tol, uint32_t cls,
                                            uint32_t i, uint32_t& t, uint32_t& aw) {
  t = a.w_taint ? (uint32_t)__popcll(taints & ~tol) : 0u;
  aw = (a.w_naff && cls != PREF_NONE) ? (uint32_t)a.pref_weights[(size_t)cls * a.Npad + i] : 0u;
}
// TaintToleration + NodeAffinity of one fitting pair, normalized by the pod's maxima over its fit set (NormalizeReduce
// with MaxNodeScore 100; reversed for the taints), weighted, int64 wrapping
__device__ __forceinline__ uint64_t pref_term(const PriorityPrefArgs& a, uint32_t t, uint32_t aw, uint32_t mt,
                                              uint32_t ma) {
  const int64_t tt = mt == 0 ? 100 : 100 - (int64_t)100 * t / mt;
  const int64_t na = ma == 0 ? 0 : (int64_t)100 * aw / ma;
  return (uint64_t)a.w_taint * (uint64_t)tt + (uint64_t)a.w_naff * (uint64_t)na;
}

// LOC's arguments (bs_upload_node_locality / bs_upload_pod_locality): the IL table the pre-pass built, each node's
// preferAvoidPods mask, each pod's class and controller bit, and the two weights.  Derived from PREF's type for the same
// reason; the ratio and preference fields are read only with RATIO and PREF.
constexpr uint32_t IMAGE_NONE = 0xffffffffu;   // BS_IMAGE_NONE
constexpr uint32_t AVOID_NONE = 0xffu;         // BS_AVOID_NONE
struct PriorityLocArgs : PriorityPrefArgs {
  const uint8_t* il;            // [classes][Npad] IL of (class, node), 0..100 (locality_class_kernel)
  const uint64_t* avoid_mask;   // [Npad] (padding 0)
  const uint32_t* loc_class;    // [P] row of il or IMAGE_NONE
  const uint8_t* avoid_bit;     // [P] 0..63 or AVOID_NONE
  uint32_t w_img, w_avoid;
};
// The pod's side of LOC: its row of the IL table (null: IL = 0) and its controller as a one-bit mask (0: none).  A
// weight of 0 skips the column, which may then be missing.
__device__ __forceinline__ void loc_pod(const PriorityLocArgs& a, uint32_t p, const uint8_t*& row, uint64_t& amask) {
  const uint32_t c = a.w_img ? a.loc_class[p] : IMAGE_NONE;
  row = c == IMAGE_NONE ? nullptr : a.il + (size_t)c * a.Npad;
  const uint32_t b = a.w_avoid ? a.avoid_bit[p] : AVOID_NONE;
  amask = b == AVOID_NONE ? 0ull : 1ull << b;
}
// w_img * IL + w_avoid * NPA of one pair, int64 wrapping: NPA is 0 when the node's annotation lists the pod's controller
__device__ __forceinline__ uint64_t loc_term(const PriorityLocArgs& a, const uint8_t* row, uint64_t amask, uint32_t i,
                                             uint64_t node_avoid) {
  const uint64_t il = row ? row[i] : 0u;
  return (uint64_t)a.w_img * il + (uint64_t)a.w_avoid * ((node_avoid & amask) ? 0u : 100u);
}

// SPREAD's arguments (bs_upload_node_spread / bs_upload_pod_spread): each node's zone, the class x node counts, each
// pod's class, and the weight.  Derived from LOC's type for the same reason; the fields of the other flags are read only
// with their flags.
constexpr uint32_t SPREAD_NONE = 0xffffffffu;   // BS_SPREAD_NONE
constexpr uint32_t ZONE_NONE = 0xffu;           // BS_ZONE_NONE
constexpr int SPREAD_ZONES = 64;                // BS_SPREAD_ZONE_MAX
struct PrioritySpreadArgs : PriorityLocArgs {
  const uint8_t* spread_zone;     // [Npad] 0..63 or ZONE_NONE (padding ZONE_NONE)
  const int32_t* spread_counts;   // [classes][Npad] (padding 0)
  const uint32_t* spread_class;   // [P] row of spread_counts or SPREAD_NONE
  uint32_t w_spread;
};
// SelectorSpread of one fitting pair (CalculateSpreadPriorityReduce): cnt = the pair's count, mn = the pod's maximum
// over its fit set, zsum / mz = the sum of the node's zone and the largest zone sum (zoned: the node has a zone).  Every operation is a binary64 rounding of its own whatever -fmad says, and the
// result is truncated toward zero.
__device__ __forceinline__ int64_t spread_score(uint32_t cnt, uint32_t mn, bool zoned, uint64_t zsum, uint64_t mz) {
  constexpr double ZW = 2.0 / 3.0;   // zoneWeighting
  double f = mn > 0 ? __dmul_rn(100.0, __ddiv_rn((double)(mn - cnt), (double)mn)) : 100.0;
  if (zoned) {
    const double zs = mz > 0 ? __dmul_rn(100.0, __ddiv_rn(__ull2double_rn(mz - zsum), __ull2double_rn(mz))) : 100.0;
    f = __dadd_rn(__dmul_rn(f, 1.0 - ZW), __dmul_rn(ZW, zs));
  }
  return __double2ll_rz(f);
}

// IPA's arguments (bs_upload_node_interpod / bs_upload_pod_interpod): the class x node raw table the IPA pre-pass
// built, each pod's class, and the weight.  Derived from SPREAD's type for the same reason; the fields of the other
// flags are read only with their flags.
constexpr uint32_t IPA_NONE = 0xffffffffu;   // BS_IPA_NONE
constexpr uint32_t TOPO_NONE = 0xffffffffu;  // BS_TOPO_NONE
constexpr int IPA_CLASS_MAX = 64;            // BS_IPA_CLASS_MAX
struct PriorityIpaArgs : PrioritySpreadArgs {
  const int64_t* ipa_raw;       // [classes][Npad] raw of (class, node) (padding 0)
  const uint32_t* ipa_class;    // [P] row of ipa_raw or IPA_NONE
  uint32_t w_ipa;
};
// InterPodAffinity of one fitting pair (CalculateInterPodAffinityPriorityReduce): raw = the pair's raw score, mn / mx =
// the pod's minimum and maximum over its fit set, both started at 0.  |raw| <= 2^47 (bsched.h), so raw - mn and
// mx - mn convert exactly; the division and the product are binary64 roundings of their own whatever -fmad says, and
// the result is truncated toward zero.
__device__ __forceinline__ int64_t ipa_score(int64_t raw, int64_t mn, int64_t mx) {
  if (mx - mn <= 0) return 0;
  return __double2ll_rz(__dmul_rn(100.0, __ddiv_rn(__ll2double_rn(raw - mn), __ll2double_rn(mx - mn))));
}

// The LOC pre-pass (priority_inst.cu image_spread_kernel, locality_class_kernel) builds the IL table once per
// change of either side or a weight; the IPA pre-pass (priority_inst.cu interpod_mass_kernel, interpod_class_kernel)
// builds the raw table once per change of either side.
constexpr int LOC_THREADS = 256;

// PREF (chosen by the host when either weight of bs_set_node_priority_weights is non-zero) adds w_taint * TT +
// w_naff * NA.  Both are normalized by the maximum raw count over the pod's fit set, and floor(100 * a / Ma) re-orders
// nodes already seen when Ma grows, so every maximum has to be known before the first pair is scored: the warp first
// sweeps the nodes once with the same fit test, keeping the largest t and a of each of its pods over the nodes that
// fit, and reduces them across its lanes.  The sweep lives in the kernel (not a [2][P] pre-pass) because its fit test
// needs the pod's requests and gate row, which the warp has already loaded for the scoring sweep.
//
// LOC (chosen by the host when either weight of bs_set_locality_weights is non-zero) adds w_img * IL + w_avoid * NPA:
// one byte of the pod's IL row per pair, read by adjacent lanes, and the node's avoid mask, shared by the warp's pods.
//
// SPREAD (chosen by the host when bs_set_spread_weight is non-zero) adds w_spread * SS.  Like PREF it needs the pod's
// maxima over its fit set before the first pair is scored, so the first sweep (one sweep for PREF, SPREAD or both)
// also keeps, per pod, the largest count (a register per lane, reduced after the sweep) and each zone's sum of counts
// over the fitting nodes (s_zs, shared memory).  A node with count 0 adds nothing to its zone, so only nodes with a
// count reach s_zs: the lanes with the same zone add theirs with __match_any_sync and __reduce_add_sync, and one lane
// of each zone adds the result with one shared atomic.  After the sweep the warp takes each pod's largest zone sum.
// haveZones needs no state of its own: it only changes the score of a fitting node with a zone, and that node makes it
// true.  A pod without selectors (SPREAD_NONE) scores 100 and reads nothing.
//
// IPA (chosen by the host when bs_set_interpod_weight is non-zero) adds w_ipa * IPA.  The pre-pass has already summed
// every bound pod's terms into one int64 raw per (class, node), so the pair reads one int64; the normalization needs
// the pod's minimum and maximum raw over its fit set, which the first sweep (shared with PREF and SPREAD) keeps per lane,
// both started at 0, and reduces across the warp into shared memory, so that they hold no register in the scoring
// sweep.  A pod without a class (IPA_NONE) scores 0 and reads nothing.
//
// LOC's, SPREAD's and IPA's kernels ask for two CTAs per SM: left to itself, ptxas gives the PREF + LOC variants up to
// 145 registers, which fits one 256-thread CTA per SM where the kernels without LOC run two.
template <int MAXL, bool RATIO, bool PREF, bool LOC = false, bool SPREAD = false, bool IPA = false>
__global__ void __launch_bounds__(PRIO_THREADS, (LOC || SPREAD || IPA) ? 2 : 0)
priority_pod_kernel(std::conditional_t<IPA, PriorityIpaArgs,
                    std::conditional_t<SPREAD, PrioritySpreadArgs,
                    std::conditional_t<LOC, PriorityLocArgs,
                                       std::conditional_t<PREF, PriorityPrefArgs,
                                                          std::conditional_t<RATIO, PriorityRatioArgs, PriorityArgs>>>>> a) {
  constexpr int WARPS = PRIO_THREADS / 32;
  __shared__ int64_t s_req[WARPS][PRIO_PPW][MAXL];
  __shared__ int64_t s_ls[WARPS][PRIO_PPW][32];
  __shared__ int32_t s_ln[WARPS][PRIO_PPW][32];
  [[maybe_unused]] const int32_t* tab = nullptr;   // RATIO: shape(util) in shared memory
  if constexpr (RATIO) {
    __shared__ int32_t s_tab[RATIO_TABLE];
    for (uint32_t k = threadIdx.x; k < (uint32_t)RATIO_TABLE; k += PRIO_THREADS) s_tab[k] = a.ratio.table[k];
    __syncthreads();
    tab = s_tab;
  }
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const uint32_t p0 = (blockIdx.x * WARPS + wid) * PRIO_PPW;
  const int L = (int)a.L;
  for (uint32_t k = lane; k < PRIO_PPW * MAXL; k += 32) {
    const uint32_t j = k / MAXL, d = k % MAXL, p = p0 + j;
    s_req[wid][j][d] = (p < a.P && d < a.L) ? a.req[(size_t)d * a.P + p] : 0;
  }
#pragma unroll
  for (int j = 0; j < PRIO_PPW; ++j) {
    s_ls[wid][j][lane] = INT64_MIN;
    s_ln[wid][j][lane] = PRIO_EMPTY;
  }
  __syncwarp();
  uint32_t rmask[PRIO_PPW];   // lanes compared: 0-3 always, scalar lanes the pod requests; 0 = no pod
  const uint32_t* grow[PRIO_PPW];
  int64_t nz_cpu[PRIO_PPW], nz_mem[PRIO_PPW], thr[PRIO_PPW];
  uint32_t nfit[PRIO_PPW];
#pragma unroll
  for (int j = 0; j < PRIO_PPW; ++j) {
    const uint32_t p = p0 + j;
    const bool ok = p < a.P;
    rmask[j] = ok ? (a.req_present[p] | 0xFu) : 0u;
    grow[j] = a.gate + (size_t)(ok ? a.fit_class[p] : 0u) * a.Wg;
    nz_cpu[j] = ok ? a.pod_nz[p] : 0;
    nz_mem[j] = ok ? a.pod_nz[(size_t)a.P + p] : 0;
    thr[j] = INT64_MIN;
    nfit[j] = 0;
  }
  [[maybe_unused]] const uint8_t* lrow[PRIO_PPW];   // LOC: the pod's IL row and controller bit
  [[maybe_unused]] uint64_t lmask[PRIO_PPW];
  if constexpr (LOC) {
#pragma unroll
    for (int j = 0; j < PRIO_PPW; ++j) {
      lrow[j] = nullptr;
      lmask[j] = 0;
      if (rmask[j]) loc_pod(a, p0 + j, lrow[j], lmask[j]);
    }
  }
  [[maybe_unused]] uint64_t ptol[PRIO_PPW];
  [[maybe_unused]] uint32_t pcls[PRIO_PPW], mt[PRIO_PPW], ma[PRIO_PPW];   // PREF: the pod's maxima over its fit set
  // SPREAD: the pod's class, its largest count and largest zone sum over its fit set
  [[maybe_unused]] uint32_t scls[PRIO_PPW], mn[PRIO_PPW];
  [[maybe_unused]] uint64_t mz[PRIO_PPW];
  [[maybe_unused]] uint64_t (*zs)[SPREAD_ZONES] = nullptr;   // SPREAD: the warp's zone sums, [PRIO_PPW][64]
  if constexpr (SPREAD) {
    __shared__ uint64_t s_zs[WARPS][PRIO_PPW][SPREAD_ZONES];
    zs = s_zs[wid];
    for (uint32_t k = lane; k < PRIO_PPW * SPREAD_ZONES; k += 32) zs[k / SPREAD_ZONES][k % SPREAD_ZONES] = 0;
#pragma unroll
    for (int j = 0; j < PRIO_PPW; ++j) {
      scls[j] = rmask[j] ? a.spread_class[p0 + j] : SPREAD_NONE;
      mn[j] = 0;
    }
    __syncwarp();
  }
  // IPA: the pod's class, and its minimum and maximum raw over its fit set ([PRIO_PPW][2], the warp's, shared memory)
  [[maybe_unused]] uint32_t icls[PRIO_PPW];
  [[maybe_unused]] int64_t (*ipm)[2] = nullptr;
  if constexpr (IPA) {
    __shared__ int64_t s_ipm[WARPS][PRIO_PPW][2];
    ipm = s_ipm[wid];
#pragma unroll
    for (int j = 0; j < PRIO_PPW; ++j) icls[j] = rmask[j] ? a.ipa_class[p0 + j] : IPA_NONE;
  }
  if constexpr (PREF || SPREAD || IPA) {
    [[maybe_unused]] int64_t imn[PRIO_PPW], imx[PRIO_PPW];   // IPA: this lane's extremes, both started at 0
    if constexpr (IPA) {
#pragma unroll
      for (int j = 0; j < PRIO_PPW; ++j) imn[j] = imx[j] = 0;
    }
    if constexpr (PREF) {
#pragma unroll
      for (int j = 0; j < PRIO_PPW; ++j) {
        const uint32_t p = p0 + j;
        ptol[j] = rmask[j] && a.w_taint ? a.prefer_tol[p] : 0;   // a column whose weight is 0 may be missing
        pcls[j] = rmask[j] && a.w_naff ? a.pref_class[p] : PREF_NONE;
        mt[j] = ma[j] = 0;
      }
    }
    // the first sweep: the fit test of the scoring sweep below, then the raw counts of the fitting nodes
    for (uint32_t base = 0; base < a.N; base += 32) {
      const uint32_t i = base + lane, w = base >> 5;
      bool g[PRIO_PPW];
      uint32_t any = 0;
#pragma unroll
      for (int j = 0; j < PRIO_PPW; ++j) {
        const uint32_t gw = rmask[j] ? grow[j][w] : 0u;
        any |= gw;
        g[j] = (gw >> lane) & 1u;
      }
      if (!any) continue;   // warp-uniform
      const uint32_t lp = a.left_present[i] | 0xFu;
#pragma unroll
      for (int d = 0; d < MAXL; ++d) {
        if (d >= L) break;
        const int64_t v = a.left[(size_t)d * a.Npad + i];
        const bool pres = (lp >> d) & 1u;
#pragma unroll
        for (int j = 0; j < PRIO_PPW; ++j)
          if (((rmask[j] >> d) & 1u) && lane_short(pres, v, s_req[wid][j][d])) g[j] = false;
      }
      if constexpr (PREF) {
        const uint64_t taints = a.w_taint ? a.prefer_taints[i] : 0;
#pragma unroll
        for (int j = 0; j < PRIO_PPW; ++j) {
          if (!g[j]) continue;
          uint32_t t, aw;
          pref_counts(a, taints, ptol[j], pcls[j], i, t, aw);
          mt[j] = max(mt[j], t);
          ma[j] = max(ma[j], aw);
        }
      }
      if constexpr (SPREAD) {
        const uint32_t z = a.spread_zone[i];   // i < Npad: padding is ZONE_NONE
#pragma unroll
        for (int j = 0; j < PRIO_PPW; ++j) {
          if (scls[j] == SPREAD_NONE) continue;   // warp-uniform
          const uint32_t cnt = g[j] ? (uint32_t)a.spread_counts[(size_t)scls[j] * a.Npad + i] : 0u;
          mn[j] = max(mn[j], cnt);
          // zone sums: one shared atomic per zone that some lane's count reaches
          const bool add = cnt != 0 && z != ZONE_NONE;
          if (!__any_sync(0xffffffffu, add)) continue;   // warp-uniform
          const uint32_t peers = __match_any_sync(0xffffffffu, add ? z : 0xffffffffu);
          if (add) {
            const uint32_t sum = __reduce_add_sync(peers, cnt);   // at most 32 x 2^24: no wrap
            if (lane == (uint32_t)(__ffs(peers) - 1)) atomicAdd((unsigned long long*)&zs[j][z], (unsigned long long)sum);
          }
        }
      }
      if constexpr (IPA) {
#pragma unroll
        for (int j = 0; j < PRIO_PPW; ++j) {
          if (!g[j] || icls[j] == IPA_NONE) continue;
          const int64_t r = a.ipa_raw[(size_t)icls[j] * a.Npad + i];
          imn[j] = min(imn[j], r);
          imx[j] = max(imx[j], r);
        }
      }
    }
    if constexpr (PREF) {
#pragma unroll
      for (int j = 0; j < PRIO_PPW; ++j) {
        mt[j] = __reduce_max_sync(0xffffffffu, mt[j]);
        ma[j] = __reduce_max_sync(0xffffffffu, ma[j]);
      }
    }
    if constexpr (SPREAD) {
      __syncwarp();
#pragma unroll
      for (int j = 0; j < PRIO_PPW; ++j) {
        mn[j] = __reduce_max_sync(0xffffffffu, mn[j]);
        uint64_t m = max(zs[j][lane], zs[j][lane + 32]);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
        mz[j] = m;
      }
    }
    if constexpr (IPA) {
#pragma unroll
      for (int j = 0; j < PRIO_PPW; ++j) {
        int64_t lo = imn[j], hi = imx[j];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          lo = min(lo, __shfl_xor_sync(0xffffffffu, lo, o));
          hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, o));
        }
        if (lane == 0) { ipm[j][0] = lo; ipm[j][1] = hi; }
      }
      __syncwarp();
    }
  }
  for (uint32_t base = 0; base < a.N; base += 32) {
    const uint32_t i = base + lane, w = base >> 5;
    bool g[PRIO_PPW];
    uint32_t any = 0;
#pragma unroll
    for (int j = 0; j < PRIO_PPW; ++j) {
      const uint32_t gw = rmask[j] ? grow[j][w] : 0u;   // the word of the padded table: bits >= N are 0
      any |= gw;
      g[j] = (gw >> lane) & 1u;
    }
    if (!any) continue;   // warp-uniform: no pod of the warp looks at these 32 nodes
    const uint32_t lp = a.left_present[i] | 0xFu;   // i < Npad: the padded tables are readable
#pragma unroll
    for (int d = 0; d < MAXL; ++d) {
      if (d >= L) break;
      const int64_t v = a.left[(size_t)d * a.Npad + i];
      const bool pres = (lp >> d) & 1u;
#pragma unroll
      for (int j = 0; j < PRIO_PPW; ++j)
        if (((rmask[j] >> d) & 1u) && lane_short(pres, v, s_req[wid][j][d])) g[j] = false;
    }
    uint32_t fw[PRIO_PPW], anyfit = 0;
#pragma unroll
    for (int j = 0; j < PRIO_PPW; ++j) {
      fw[j] = __ballot_sync(0xffffffffu, g[j]);
      anyfit |= fw[j];
    }
    if (!anyfit) continue;
    const int64_t c_cpu = a.alloc[i], c_mem = a.alloc[(size_t)a.Npad + i];
    const int64_t n_cpu = a.node_nz[i], n_mem = a.node_nz[(size_t)a.Npad + i];
    [[maybe_unused]] uint64_t navoid = 0;   // LOC: the node's preferAvoidPods mask
    if constexpr (LOC) navoid = a.w_avoid ? a.avoid_mask[i] : 0;
    [[maybe_unused]] uint32_t nzone = ZONE_NONE;   // SPREAD: the node's zone
    if constexpr (SPREAD) nzone = a.spread_zone[i];
    [[maybe_unused]] uint32_t rnum[PRIO_PPW], rden[PRIO_PPW];   // RATIO: the weighted sum and weight sum of each pod's average
    if constexpr (RATIO) {
#pragma unroll
      for (int j = 0; j < PRIO_PPW; ++j) { rnum[j] = a.ratio.num0; rden[j] = a.ratio.den0; }
      const uint32_t ap = a.node_alloc_present[i], rp = a.node_req_present[i];
#pragma unroll
      for (int d = 0; d < MAXL; ++d) {
        const uint32_t wd = a.ratio.lane_w[d];
        if (!wd) continue;   // uniform; lanes 3 and >= L weigh 0
        // capacity and the node's term: cpu / memory from the non-zero column; lane 2 and the scalar lanes from the
        // node table, 0 for a key the node lacks
        int64_t c, rn;
        if (d == LANE_CPU) { c = c_cpu; rn = n_cpu; }
        else if (d == LANE_MEM) { c = c_mem; rn = n_mem; }
        else {
          c = (d < 4 || ((ap >> d) & 1u)) ? a.alloc[(size_t)d * a.Npad + i] : 0;
          rn = (d < 4 || ((rp >> d) & 1u)) ? a.node_requested[(size_t)d * a.Npad + i] : 0;
        }
#pragma unroll
        for (int j = 0; j < PRIO_PPW; ++j) {
          if (!fw[j]) continue;   // warp-uniform
          const int64_t rq = d == LANE_CPU ? nz_cpu[j] : d == LANE_MEM ? nz_mem[j]
                                                       : (((rmask[j] >> d) & 1u) ? s_req[wid][j][d] : 0);
          ratio_accumulate(ratio_lane_score(tab, (int64_t)((uint64_t)rn + (uint64_t)rq), c), wd, rnum[j], rden[j]);
        }
      }
    }
#pragma unroll
    for (int j = 0; j < PRIO_PPW; ++j) {
      if (!fw[j]) continue;   // warp-uniform
      int64_t s = g[j] ? pair_score(n_cpu + nz_cpu[j], c_cpu, n_mem + nz_mem[j], c_mem, a.w) : INT64_MIN;
      if constexpr (RATIO)
        if (g[j]) s = (int64_t)((uint64_t)s + ratio_term(a.ratio.weight, rnum[j], rden[j]));
      if constexpr (PREF)
        if (g[j]) {
          uint32_t t, aw;
          pref_counts(a, a.w_taint ? a.prefer_taints[i] : 0, ptol[j], pcls[j], i, t, aw);
          s = (int64_t)((uint64_t)s + pref_term(a, t, aw, mt[j], ma[j]));
        }
      if constexpr (LOC)
        if (g[j]) s = (int64_t)((uint64_t)s + loc_term(a, lrow[j], lmask[j], i, navoid));
      if constexpr (SPREAD)
        if (g[j]) {
          int64_t ss = 100;
          if (scls[j] != SPREAD_NONE) {
            const bool zoned = nzone != ZONE_NONE;   // a fitting node with a zone: haveZones holds
            ss = spread_score((uint32_t)a.spread_counts[(size_t)scls[j] * a.Npad + i], mn[j], zoned,
                              zoned ? zs[j][nzone] : 0ull, mz[j]);
          }
          s = (int64_t)((uint64_t)s + (uint64_t)a.w_spread * (uint64_t)ss);
        }
      if constexpr (IPA)
        if (g[j] && icls[j] != IPA_NONE) {
          const int64_t is = ipa_score(a.ipa_raw[(size_t)icls[j] * a.Npad + i], ipm[j][0], ipm[j][1]);
          s = (int64_t)((uint64_t)s + (uint64_t)a.w_ipa * (uint64_t)is);
        }
      const uint32_t cb = __ballot_sync(0xffffffffu, g[j] && (nfit[j] < a.K || s > thr[j]));
      if (cb) thr[j] = topk_insert<int64_t>(s_ls[wid][j], s_ln[wid][j], a.K, cb, s, (int32_t)base, lane);
      nfit[j] += __popc(fw[j]);
    }
  }
#pragma unroll
  for (int j = 0; j < PRIO_PPW; ++j) {
    const uint32_t p = p0 + j;
    if (p < a.P && lane < a.K) {
      const int32_t n = s_ln[wid][j][lane];
      a.out_node[(size_t)p * a.K + lane] = n == PRIO_EMPTY ? -1 : n;
      a.out_score[(size_t)p * a.K + lane] = n == PRIO_EMPTY ? INT64_MIN : s_ls[wid][j][lane];
    }
  }
}

// The builds of priority_pod_kernel: one per lane bound MAXL = 5, 9, 16 and mask of the terms below, 96 in all.  The host
// sets a term's bit when its weight is non-zero; `a` is read as the build's argument type (PriorityArgs without any
// term, PriorityRatioArgs with RATIO alone, PriorityPrefArgs with PREF, PriorityLocArgs with LOC, PrioritySpreadArgs
// with SPREAD, all of it with IPA).
constexpr uint32_t PRIO_RATIO = 1, PRIO_PREF = 2, PRIO_LOC = 4, PRIO_SPREAD = 8, PRIO_IPA = 16;
// priority_inst.cu, one slice per (MAXL, IPA bit): launches the build of lane bound MAXL for `terms`, whose IPA bit is
// IPA (engine.cu's launch_priority picks the slice)
template <int MAXL, uint32_t IPA>
void launch_priority_slice(uint32_t terms, uint32_t grid, const PriorityIpaArgs& a, cudaStream_t s);
// the LOC pre-pass: scaled[n_images] from the bit rows and sizes, then il[n_classes][Npad]; 2 launches
cudaError_t launch_locality_prepass(const uint32_t* bits, const int64_t* size, int64_t* scaled, uint32_t n_images,
                                    const uint32_t* class_offset, const uint32_t* class_images, uint8_t* il,
                                    uint32_t n_classes, uint32_t n_nodes, uint32_t Npad, cudaStream_t s);
// The IPA pre-pass over device copies of the bs_interpod_nodes / bs_interpod_pods columns.  term_off[t]: the first
// (term, value) slot of term t; ms[slots][2]: M and S, zeroed by the caller.  With mass, the bound pods are summed into
// ms first (1 launch); then raw[n_pod_classes][Npad] (1 launch).
struct InterpodClasses {
  const uint32_t* offset;   // [n_classes + 1]
  const uint32_t* term;
  const int32_t* own;
  const uint8_t* match;
  uint32_t n_classes;
};
cudaError_t launch_interpod_prepass(bool mass, const uint32_t* topo, const uint32_t* term_key, const uint32_t* term_off,
                                    const uint32_t* bound_node, const uint32_t* bound_class, uint32_t n_bound,
                                    const InterpodClasses& bound, const InterpodClasses& pods, int64_t* ms,
                                    int64_t* raw, uint32_t n_nodes, uint32_t Npad, cudaStream_t s);

}  // namespace bsk
