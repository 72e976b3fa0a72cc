// replay.cuh — multi-round admission on the device (SURVEY.md §8(f) row 4).
//
// The reference schedules ONE pod per cycle against mutable caches: PreFilter reads the live
// PodGroup state and the live snapshot (core.go:88-167), the pod is assumed onto a node
// (NodeInfo.AddPod debits `requested`), Permit records the match and may flip the group to
// Scheduled (core.go:268-309).  Every step depends on the previous one, so the queue is walked by
// ONE persistent CTA (256 threads: registers to spare, cheap barriers); the parallelism is inside
// a step:
//   node state         next to the reference-format columns it returns, the kernel keeps the
//                      residuals singleNodeResource would compute (percent 1.0 and 0.7, int64,
//                      zero for absent scalar keys), the key mask and one checkFit bit per
//                      representative class; a step reads them with 16-byte loads, four consecutive
//                      nodes per thread, and only the assumed node's row is rewritten;
//   findMaxPG          the group table is cut into <= 1024 buckets whose merged states (the
//                      order-insensitive merge of kernels.cuh) sit in shared memory; a changed group
//                      costs one warp one bucket, the answer is one block reduction, and it is
//                      recomputed only after some group changed;
//   cluster check      blocks of 1024 nodes: serial prefix over a thread's four nodes, warp-shuffle
//                      scan of the thread totals, running carry, every prefix tested, block-wide OR
//                      (the reference returns true at the first satisfying prefix == some prefix
//                      satisfies).  Blocks are not rescanned blindly: per (representative class,
//                      percent, block) the block total, key set and per-lane maximum of the in-block
//                      prefix are cached (one node changes per step, so one block goes stale); a
//                      block whose carry + maximum stays below the need on a compared lane cannot
//                      hold a satisfying prefix and is skipped, the others are scanned exactly, in
//                      order.  A stale first block is scanned exactly before anything else: where
//                      the cluster has room the need is met there;
//   node choice        bs_replay (SCORED = false): first node in list order where the pod fits, the
//                      stand-in for the upstream filter/selectHost the oracle uses too.
//                      bs_replay_priority (SCORED = true): every fitting node is scored with
//                      pair_score on the live non-zero column and the best one wins (score
//                      descending, then index ascending): each thread keeps the best of its four
//                      nodes over the sweep, one block reduction picks the winner.  RATIO (a non-zero
//                      bs_set_ratio_priority weight) adds the RequestedToCapacityRatio term over the
//                      live `requested` and key mask (lanes >= 2) and the live non-zero column.  LOC (a
//                      non-zero bs_set_locality_weights weight) adds ImageLocality and NodePreferAvoidPods,
//                      which the walk does not change: the round's IL table and avoid masks.  In both,
//                      requests only grow `requested`, so a leading run of nodes no pod of the table
//                      can ever fit again (or that is skipped) is remembered and not rescanned; such
//                      a node never fits, so it never scores either;
//   assume + Permit    a handful of stores by the first lanes (SCORED: the chosen node's live
//                      non-zero column grows by the pod's, NodeInfo.AddPod's nonzeroRequest).
// Mutable state lives in scratch copies (requested, pod_count, req_present, matched, group flags,
// representative class, MinResources, the live non-zero column); the uploaded tables are untouched.
#pragma once
#include "kernels.cuh"

#include <type_traits>

namespace bsk {

constexpr int REPLAY_THREADS = 256;
constexpr int REPLAY_WARPS = REPLAY_THREADS / 32;
constexpr int REPLAY_NPT = 4;                                  // consecutive nodes per thread
constexpr int REPLAY_BLOCK = REPLAY_THREADS * REPLAY_NPT;      // nodes per scan block
constexpr int REPLAY_MAX_BUCKETS = 1024;                       // findMaxPG buckets
constexpr int REPLAY_MAX_BLOCKS = REPLAY_BLOCK;                // blocks the summary cache can index
constexpr int REPLAY_MAX_CLASSES = 32;                         // representative classes with a checkFit bit

// node status bits of the compact table
constexpr uint32_t RN_VISITED = 1;    // in the list and not skipped (core.go:606-617)
constexpr uint32_t RN_TAINTS_OK = 2;  // info.Taints() did not fail (:639)

struct ReplayArgs {
  NodeTab nt;                 // requested / pod_count / req_present point at the SCRATCH copies
  int64_t* requested;         // [L][Npad] scratch (same memory as nt.requested)
  int32_t* pod_count;
  uint32_t* req_present;
  int64_t* left[2];           // [L][Npad] residual at percent 1.0 / 0.7 (class-free), 0 for absent keys
  uint32_t* both;             // [Npad] scalar keys present in allocatable AND requested (:662-666)
  uint32_t* fitmask;          // [Npad] bit c: checkFit(class c); null when n_rep > 32
  uint8_t* nstat;             // [Npad] RN_*
  PodTab pt;
  const uint64_t* rsel;       // representative-class tables (every pod's (sel, tol) is one of them)
  const uint64_t* rtol;
  const uint32_t* raff;       // affinity class of each representative class (BS_AFF_NONE: none)
  uint32_t n_rep;
  uint32_t cache_ok;          // block summaries usable: sums stay below 2^62 and the scratch exists (host)
  int64_t* blk_sum;           // [2*n_rep][n_blocks][MAXL] block totals
  int64_t* blk_max;           // [2*n_rep][n_blocks][MAXL] max in-block prefix per lane
  uint32_t* blk_keys;         // [2*n_rep][n_blocks]       scalar keys seen in the block
  const uint32_t* min_member;
  const uint32_t* scheduled;
  uint32_t* matched;          // scratch
  uint8_t* gflags;            // scratch
  uint32_t* grc;              // scratch: representative class per group
  int64_t* min_res;           // scratch [L][G]
  uint32_t* mrpres;           // scratch
  uint32_t G;
  const uint32_t* queue;      // pod indices in pop order, or null: 0..n_queue-1
  uint32_t n_queue;
  uint8_t* prefilter;         // [n_queue]
  int32_t* node;              // [n_queue]
  uint8_t* ready;             // [n_queue]
  int32_t* status;            // [0]: findMaxPG would have divided by zero (core.go:716); [1] the final `lo` of
                              // the dead-node skip, [2] `monotone` (bs_replay_shape)
  // bs_replay_priority only (SCORED): the live node column, the pod column and the weights of the node choice
  int64_t* nz_live;           // [2][Npad] scratch copy of the uploaded node column
  const int64_t* pod_nz;      // [2][P]
  ScoreWeights w;
  RatioSetting ratio;         // RATIO only
};
// LOC's arguments (priority.cuh PriorityLocArgs): a derived type, so that the kernels without the terms keep theirs
struct ReplayLocArgs : ReplayArgs {
  const uint8_t* il;            // [classes][Npad]
  const uint64_t* avoid_mask;   // [Npad]
  const uint32_t* loc_class;    // [P]
  const uint8_t* avoid_bit;     // [P]
  uint32_t w_img, w_avoid;
};

template <int MAXL>
struct ReplaySmem {
  MaxState bucket[REPLAY_MAX_BUCKETS];   // merged findMaxPG state of each bucket of groups
  MaxState part[32];
  uint32_t valid[2 * REPLAY_MAX_CLASSES][REPLAY_MAX_BLOCKS / 32];   // block summaries that are current
  uint8_t cand[REPLAY_MAX_BLOCKS];       // blocks that may hold a satisfying prefix
  int64_t woff[REPLAY_WARPS][MAXL];      // carry + exclusive warp offsets of the current block of nodes
  int64_t wmax[REPLAY_WARPS][MAXL];
  uint32_t wkeys[REPLAY_WARPS];
  int64_t carry[MAXL];                   // running total in front of / after the current block
  uint32_t carry_keys;
  int64_t req[2][MAXL];                  // getPodResourceRequire of the current / next pod
  int64_t need[MAXL];
  int64_t min_req[4];                    // smallest request of any pod of the table, fixed lanes
  int32_t monotone;                      // no pod has a negative fixed-lane request: residuals only shrink
  int32_t first[2];                      // chosen node, one slot per step parity
  int32_t max_group;
  int32_t panic;
};

// compareResourceAndRequire (core.go:672-699): `left` in registers, `req` in shared memory
template <int MAXL>
__device__ __forceinline__ bool compare_lanes(const int64_t (&left)[MAXL], uint32_t lkeys, const int64_t* req,
                                              uint32_t rkeys) {
  bool ok = (left[LANE_MEM] >= req[LANE_MEM]) & (left[LANE_CPU] >= req[LANE_CPU]) &
            (left[LANE_EPH] >= req[LANE_EPH]) & (left[LANE_PODS] >= req[LANE_PODS]);
#pragma unroll
  for (int d = 4; d < MAXL; ++d) {
    const uint32_t bit = 1u << d;
    if (rkeys & bit) ok &= (lkeys & bit) ? (req[d] <= left[d]) : (req[d] == 0);   // :686-697
  }
  return ok;
}

// Inclusive scan over the 1024 items of a block, four consecutive items per thread (sum of v,
// OR of keys).  use_carry adds sm.carry in front; update_carry leaves the total (carry included)
// in sm.carry.  Two barriers inside; the caller puts one more before the next call.
template <int MAXL>
__device__ __forceinline__ void block_scan(ReplaySmem<MAXL>& sm, int64_t (&v)[REPLAY_NPT][MAXL],
                                           uint32_t (&keys)[REPLAY_NPT], bool use_carry, bool update_carry) {
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int k = 1; k < REPLAY_NPT; ++k) {
#pragma unroll
    for (int d = 0; d < MAXL; ++d) v[k][d] += v[k - 1][d];
    keys[k] |= keys[k - 1];
  }
  int64_t tot[MAXL];
  uint32_t tk = keys[REPLAY_NPT - 1];
#pragma unroll
  for (int d = 0; d < MAXL; ++d) tot[d] = v[REPLAY_NPT - 1][d];
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
#pragma unroll
    for (int d = 0; d < MAXL; ++d) {
      const int64_t t = __shfl_up_sync(0xffffffffu, tot[d], o);
      if ((int)lane >= o) tot[d] += t;
    }
    const uint32_t k = __shfl_up_sync(0xffffffffu, tk, o);
    if ((int)lane >= o) tk |= k;
  }
  if (lane == 31) {
#pragma unroll
    for (int d = 0; d < MAXL; ++d) sm.woff[wid][d] = tot[d];
    sm.wkeys[wid] = tk;
  }
  __syncthreads();
  if (wid == 0) {
    int64_t x[MAXL];
#pragma unroll
    for (int d = 0; d < MAXL; ++d) x[d] = lane < REPLAY_WARPS ? sm.woff[lane][d] : 0;
    uint32_t xk = lane < REPLAY_WARPS ? sm.wkeys[lane] : 0u;
#pragma unroll
    for (int o = 1; o < REPLAY_WARPS; o <<= 1) {
#pragma unroll
      for (int d = 0; d < MAXL; ++d) {
        const int64_t t = __shfl_up_sync(0xffffffffu, x[d], o);
        if ((int)lane >= o) x[d] += t;
      }
      const uint32_t k = __shfl_up_sync(0xffffffffu, xk, o);
      if ((int)lane >= o) xk |= k;
    }
    // carry + exclusive offset of each warp, in place; the last warp's lane holds the total
    const uint32_t ck = use_carry ? sm.carry_keys : 0u;
    uint32_t exk = __shfl_up_sync(0xffffffffu, xk, 1);
    if (lane == 0) exk = 0;
#pragma unroll
    for (int d = 0; d < MAXL; ++d) {
      const int64_t c = use_carry ? sm.carry[d] : 0;
      int64_t ex = __shfl_up_sync(0xffffffffu, x[d], 1);
      if (lane == 0) ex = 0;
      if (lane < REPLAY_WARPS) sm.woff[lane][d] = c + ex;
      x[d] += c;
    }
    if (lane < REPLAY_WARPS) sm.wkeys[lane] = ck | exk;
    __syncwarp();
    if (update_carry && lane == REPLAY_WARPS - 1) {
#pragma unroll
      for (int d = 0; d < MAXL; ++d) sm.carry[d] = x[d];
      sm.carry_keys = ck | xk;
    }
  }
  __syncthreads();
  // what lies in front of this thread: the warp offset + the lanes below
  uint32_t fk = __shfl_up_sync(0xffffffffu, tk, 1);
  fk = (lane ? fk : 0u) | sm.wkeys[wid];
#pragma unroll
  for (int d = 0; d < MAXL; ++d) {
    const int64_t front = sm.woff[wid][d] + (tot[d] - v[REPLAY_NPT - 1][d]);
#pragma unroll
    for (int k = 0; k < REPLAY_NPT; ++k) v[k][d] += front;
  }
#pragma unroll
  for (int k = 0; k < REPLAY_NPT; ++k) keys[k] |= fk;
}

template <int MAXL, bool SCORED, bool RATIO = false, bool LOC = false>
__global__ void __launch_bounds__(REPLAY_THREADS, 1) replay_kernel(std::conditional_t<LOC, ReplayLocArgs, ReplayArgs> a) {
  static_assert(SCORED || !RATIO, "the ratio term belongs to the scored node choice");
  static_assert(SCORED || !LOC, "the locality terms belong to the scored node choice");
  __shared__ ReplaySmem<MAXL> sm;
  __shared__ int32_t s_tab[RATIO_TABLE];   // RATIO: shape(util)
  const uint32_t tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const uint32_t N = a.nt.N, Npad = a.nt.Npad, G = a.G, P = a.pt.P;
  const uint32_t L = a.nt.L;
  const uint32_t C = a.n_rep;
  const uint32_t NBLK = (N + REPLAY_BLOCK - 1) / REPLAY_BLOCK;
  const bool use_mask = a.fitmask != nullptr;
  const bool use_cache = a.cache_ok && use_mask && NBLK >= 1 && NBLK <= (uint32_t)REPLAY_MAX_BLOCKS;

  GroupTab gt{};
  gt.min_member = a.min_member; gt.scheduled = a.scheduled; gt.matched = a.matched;
  gt.flags = a.gflags; gt.min_res = a.min_res; gt.min_res_present = a.mrpres; gt.rep_class = a.grc;
  gt.G = G; gt.L = L;
  GroupEff ge{};
  ge.flags = a.gflags; ge.min_res = a.min_res; ge.min_res_present = a.mrpres; ge.rep_class = a.grc;

  // ---- compact node state: residuals at both percents (:647-668), key mask, checkFit bits ----
  for (uint32_t i = tid; i < Npad; i += REPLAY_THREADS) {
    uint32_t st = 0, both = 0, fm = 0;
    if (i < N) {
      const uint8_t f = a.nt.flags[i];
      if (!node_skipped(f)) st |= RN_VISITED;
      if (!(f & BS_NODE_TAINTS_ERR)) st |= RN_TAINTS_OK;
      both = a.nt.alloc_present[i] & a.nt.req_present[i] & ~0xFu;
      for (uint32_t d = 0; d < L; ++d) {
        const bool present = d < 4 || ((both >> d) & 1u);
        int64_t sub = a.nt.requested[(size_t)d * Npad + i];
        if (d == LANE_PODS && sub == 0) sub = a.nt.pod_count[i];     // :650-653
        const int64_t cap = a.nt.alloc[(size_t)d * Npad + i];
        a.left[0][(size_t)d * Npad + i] = present ? scale_f32(cap, 1.0f) - sub : 0;
        a.left[1][(size_t)d * Npad + i] = present ? scale_f32(cap, 0.7f) - sub : 0;
      }
      if (use_mask) {
        const uint64_t lb = a.nt.label[i], tn = a.nt.taint[i];
        for (uint32_t c = 0; c < C; ++c)
          if (check_fit(lb, tn, a.rsel[c], a.rtol[c]) && aff_ok(a.nt, a.raff[c], i)) fm |= 1u << c;
      }
    } else {
      for (uint32_t d = 0; d < L; ++d) { a.left[0][(size_t)d * Npad + i] = 0; a.left[1][(size_t)d * Npad + i] = 0; }
    }
    a.nstat[i] = (uint8_t)st;
    a.both[i] = both;
    if (use_mask) a.fitmask[i] = fm;
  }
  // ---- findMaxPG buckets: S consecutive groups each, at most 1024 of them ----
  const uint32_t per = (G + 32u * REPLAY_MAX_BUCKETS - 1) / (32u * REPLAY_MAX_BUCKETS);
  const uint32_t S = 32u * (per ? per : 1u);
  const uint32_t NB = (G + S - 1) / S;
  auto bucket_compute = [&](uint32_t b) {   // by one whole warp
    MaxState v = max_state_empty();
    const uint32_t g0 = b * S;
    for (uint32_t j = lane; j < S; j += 32) {
      const uint32_t i = g0 + j;
      if (i < G) v = max_state_merge(v, max_state_of(gt, ge, i));
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) v = max_state_merge(v, max_state_shfl_xor(v, o));
    if (lane == 0) sm.bucket[b] = v;
  };
  for (uint32_t b = wid; b < NB; b += REPLAY_WARPS) bucket_compute(b);
  bool max_dirty = true;     // uniform: a group changed since the last reduction
  int32_t max_group = -1;    // uniform copy of the last findMaxPG result

  // ---- smallest fixed-lane request of the table; are requests non-negative? ----
  {
    int64_t mn[4] = {INT64_MAX, INT64_MAX, INT64_MAX, INT64_MAX};
    for (uint32_t p = tid; p < P; p += REPLAY_THREADS)
#pragma unroll
      for (int d = 0; d < 4; ++d) mn[d] = min(mn[d], a.pt.req[(size_t)d * P + p]);
#pragma unroll
    for (int d = 0; d < 4; ++d) {
#pragma unroll
      for (int o = 16; o; o >>= 1) mn[d] = min(mn[d], __shfl_xor_sync(0xffffffffu, mn[d], o));
      if (lane == 0) sm.woff[wid][d] = mn[d];
    }
    __syncthreads();
    if (tid < 4) {
      int64_t m = INT64_MAX;
      for (int w = 0; w < REPLAY_WARPS; ++w) m = min(m, sm.woff[w][tid]);
      sm.min_req[tid] = m;
    }
    __syncthreads();
    if (tid == 0) sm.monotone = (sm.min_req[LANE_CPU] >= 0 && sm.min_req[LANE_MEM] >= 0 && sm.min_req[LANE_EPH] >= 0) ? 1 : 0;
  }
  for (uint32_t k = tid; k < 2u * REPLAY_MAX_CLASSES * (REPLAY_MAX_BLOCKS / 32); k += REPLAY_THREADS) (&sm.valid[0][0])[k] = 0;

  // pod columns of the NEXT step are fetched one step ahead (the walk is latency-bound)
  // SCORED: the pod's non-zero pair (cpu, memory), one slot per step parity like sm.req; a separate array, so that the
  // first-fit kernel's shared memory stays as it is
  __shared__ int64_t s_pod_nz[2][2];
  struct PodRow { uint32_t p; int32_t g; uint8_t pf; uint32_t keys, rc; };
  auto load_row = [&](uint32_t qi, int slot) {
    PodRow r;
    r.p = a.queue ? a.queue[qi] : qi;
    r.g = a.pt.gid[r.p];
    r.pf = a.pt.flags[r.p];
    const uint32_t ppres = a.pt.req_present[r.p];
    r.keys = ppres & ~0xFu;
    r.rc = a.pt.rep_class[r.p];
    if constexpr (SCORED)
      if (tid < 2) s_pod_nz[slot][tid] = a.pod_nz[(size_t)tid * P + r.p];
    if (tid < L)   // getPodResourceRequire (core.go:761-772): the packer summed the containers
      sm.req[slot][tid] = (tid < 4 || ((ppres >> tid) & 1u)) ? a.pt.req[(size_t)tid * P + r.p] : 0;
    return r;
  };
  if constexpr (RATIO)
    for (uint32_t k = tid; k < (uint32_t)RATIO_TABLE; k += REPLAY_THREADS) s_tab[k] = a.ratio.table[k];
  if (tid == 0) { sm.first[0] = 0x7fffffff; sm.first[1] = 0x7fffffff; sm.panic = 0; }
  if (tid < MAXL) { sm.req[0][tid] = 0; sm.req[1][tid] = 0; sm.need[tid] = 0; }
  __syncthreads();
  PodRow nx{};
  if (a.n_queue) nx = load_row(0, 0);
  __syncthreads();
  const bool monotone = sm.monotone != 0;
  uint32_t lo = 0;   // uniform: nodes before `lo` can never host a pod of this table again

  // The four consecutive nodes base + 4*tid .. of a block: residual lanes at percent index pi
  // (class-free), key masks, and per node (bit k): visited, Taints() ok, checkFit of class rc.
  auto load_quad = [&](uint32_t base, int pi, uint32_t rc, uint64_t sel, uint64_t tol, int64_t (&v)[REPLAY_NPT][MAXL],
                       uint32_t (&keys)[REPLAY_NPT], uint32_t& vis, uint32_t& tok, uint32_t& fit) {
    const uint32_t i0 = base + REPLAY_NPT * tid;
    vis = 0; tok = 0; fit = 0;
    if (i0 < Npad) {
      const uint32_t st4 = *reinterpret_cast<const uint32_t*>(a.nstat + i0);
      const uint4 k4 = *reinterpret_cast<const uint4*>(a.both + i0);
      keys[0] = k4.x; keys[1] = k4.y; keys[2] = k4.z; keys[3] = k4.w;
#pragma unroll
      for (int d = 0; d < MAXL; ++d) {
        if ((uint32_t)d < L) {
          const longlong2* src = reinterpret_cast<const longlong2*>(a.left[pi] + (size_t)d * Npad + i0);
          const longlong2 x = src[0], y = src[1];
          v[0][d] = x.x; v[1][d] = x.y; v[2][d] = y.x; v[3][d] = y.y;
        } else {
          v[0][d] = 0; v[1][d] = 0; v[2][d] = 0; v[3][d] = 0;
        }
      }
      if (use_mask) {
        const uint4 f4 = *reinterpret_cast<const uint4*>(a.fitmask + i0);
        fit = ((f4.x >> rc) & 1u) | (((f4.y >> rc) & 1u) << 1) | (((f4.z >> rc) & 1u) << 2) | (((f4.w >> rc) & 1u) << 3);
      } else {
#pragma unroll
        for (int k = 0; k < REPLAY_NPT; ++k)
          if (i0 + k < N && check_fit(a.nt.label[i0 + k], a.nt.taint[i0 + k], sel, tol) && aff_ok(a.nt, a.raff[rc], i0 + k))
            fit |= 1u << k;
      }
#pragma unroll
      for (int k = 0; k < REPLAY_NPT; ++k) {
        const uint32_t s = (st4 >> (8 * k)) & 0xffu;
        if (s & RN_VISITED) vis |= 1u << k;
        if (s & RN_TAINTS_OK) tok |= 1u << k;
      }
    } else {
#pragma unroll
      for (int k = 0; k < REPLAY_NPT; ++k) {
        keys[k] = 0;
#pragma unroll
        for (int d = 0; d < MAXL; ++d) v[k][d] = 0;
      }
    }
  };

  for (uint32_t qi = 0; qi < a.n_queue; ++qi) {
    const PodRow cur = nx;
    const int par = (int)(qi & 1u);
    if (qi + 1 < a.n_queue) nx = load_row(qi + 1, par ^ 1);
    if (tid == 0) sm.first[par ^ 1] = 0x7fffffff;   // read last in step qi-1, used next in step qi+1
    const int32_t g = cur.g;
    const uint8_t pf = cur.pf;
    const uint32_t req_keys = cur.keys;
    const int64_t* req = sm.req[par];

    uint8_t code = BS_PF_PASS;
    // ---- PreFilter against live state (core.go:88-167) ----
    do {
      if (g == BS_GID_NONE) break;                                   // :90-93
      if (pf & BS_POD_PERMITTED_RECENTLY) break;                     // :95-98
      if (g < 0 || (uint32_t)g >= G) { code = BS_PF_ERR_NOT_FOUND; break; }   // :100-103
      const uint8_t gf = a.gflags[g];
      if (gf & BS_GROUP_DENIED) { code = BS_PF_ERR_DENIED; break; }  // :105-110
      // fillOccupiedObj :486-493 — the first pod to arrive becomes the representative
      const bool take_pod = !(gf & BS_GROUP_HAS_POD), take_res = !(gf & BS_GROUP_HAS_MINRES);
      if (take_pod || take_res) {
        __syncthreads();   // every thread has read the group's flags before they change
        if (take_res && tid < L) a.min_res[(size_t)tid * G + g] = req[tid];
        if (tid == 0) {
          uint8_t nf = gf;
          if (take_pod) { nf |= BS_GROUP_HAS_POD; a.grc[g] = cur.rc; }
          if (take_res) { nf |= BS_GROUP_HAS_MINRES; a.mrpres[g] = req_keys; }
          a.gflags[g] = nf;
        }
        __syncthreads();
        if (take_pod) {
          if (wid == REPLAY_WARPS - 1) bucket_compute((uint32_t)g / S);
          max_dirty = true;
        }
      }
      if (pf & BS_POD_OCC_NOREFS) { code = BS_PF_ERR_OCCUPIED_NOREFS; break; }     // :494-503
      if (pf & BS_POD_OCC_MISMATCH) { code = BS_PF_ERR_OCCUPIED; break; }     // :504-511
      // findMaxPG :120 (re-reduced only when some group changed)
      if (max_dirty) {
        __syncthreads();   // bucket states written by the updating warp are visible
        MaxState mv = max_state_empty();
        for (uint32_t b = tid; b < NB; b += REPLAY_THREADS) mv = max_state_merge(mv, sm.bucket[b]);
        mv = max_state_block_reduce(mv, sm.part);
        if (tid == 0) {
          int32_t w = -1;
          if (mv.any) {
            uint32_t winner = mv.c0;
            if (mv.c0_flags & 1u) {
              if (mv.zgood != 0xffffffffu) winner = mv.zgood;
              else if (mv.zlast != 0) winner = mv.zlast - 1;
            }
            w = (int32_t)winner;
          }
          sm.max_group = w;
          sm.panic = (int32_t)mv.panic;
        }
        __syncthreads();
        max_group = sm.max_group;
        max_dirty = false;
        if (sm.panic) break;
      }
      const int32_t m = max_group;
      if (m < 0) break;                                              // :127-130
      const uint32_t matched_m = a.matched[m];
      const bool case_a = matched_m == 0;                            // :134-147
      if (!case_a && m == g) break;                                  // :150-155
      // need: getPreAllocatedResource (core.go:774-793) of this group (case A) or of the max
      // group plus the pod's own request (:157-159); one lane per thread
      const uint32_t gi = case_a ? (uint32_t)g : (uint32_t)m;
      const int64_t mm = (int64_t)a.min_member[gi];
      const int64_t not_finished = case_a ? mm - (int64_t)a.scheduled[gi] : mm - (int64_t)matched_m;   // :778-783
      const bool adds = not_finished > 0 && (a.gflags[gi] & BS_GROUP_HAS_MINRES);                       // :784-788
      const uint32_t mr_keys = adds ? a.mrpres[gi] : 0u;
      const uint32_t need_keys = mr_keys | (case_a ? 0u : req_keys);
      if (tid < L) {
        int64_t val = 0;
        if (adds && (tid < 4 || ((mr_keys >> tid) & 1u)))
          val = (int64_t)((uint64_t)a.min_res[(size_t)tid * G + gi] * (uint64_t)not_finished);
        if (tid == LANE_PODS && val == 0) val = mm + 1;              // :789-791
        if (!case_a && (tid < 4 || ((req_keys >> tid) & 1u))) val += req[tid];
        sm.need[tid] = val;
      }
      const uint32_t rc = a.grc[gi];
      const int pi = case_a ? 0 : 1;
      const uint32_t ci = rc * 2u + (uint32_t)pi;
      const uint64_t sel = a.rsel[rc], tol = a.rtol[rc];
      __syncthreads();

      // singleNodeResource of this thread's four nodes (:619): zeros when unfit (:639-645) or skipped
      auto node_terms = [&](uint32_t base, int64_t (&v)[REPLAY_NPT][MAXL], uint32_t (&keys)[REPLAY_NPT]) -> uint32_t {
        uint32_t vis, tok, fit;
        load_quad(base, pi, rc, sel, tol, v, keys, vis, tok, fit);
        const uint32_t act = vis & tok & fit;
#pragma unroll
        for (int k = 0; k < REPLAY_NPT; ++k)
          if (!((act >> k) & 1u)) {
            keys[k] = 0;
#pragma unroll
            for (int d = 0; d < MAXL; ++d) v[k][d] = 0;
          }
        return vis;
      };
      // every prefix ending in the block against the need (:621-627); ends with a barrier
      auto exact_block = [&](uint32_t base, bool use_carry, bool update_carry) -> bool {
        int64_t v[REPLAY_NPT][MAXL];
        uint32_t keys[REPLAY_NPT];
        const uint32_t vis = node_terms(base, v, keys);
        block_scan<MAXL>(sm, v, keys, use_carry, update_carry);
        bool ok = false;
#pragma unroll
        for (int k = 0; k < REPLAY_NPT; ++k)
          ok |= ((vis >> k) & 1u) && compare_lanes<MAXL>(v[k], keys[k], sm.need, need_keys);
        return __syncthreads_or(ok ? 1 : 0) != 0;
      };

      // compareClusterResourceAndRequire :595-632 — true iff some visited prefix satisfies the need
      bool enough = false;
      if (!use_cache) {
        for (uint32_t base = 0; base < N && !enough; base += REPLAY_BLOCK) enough = exact_block(base, base != 0, true);
      } else {
        const bool b0_cached = (sm.valid[ci][0] & 1u) != 0;
        if (!b0_cached) enough = exact_block(0, false, false);
        if (!enough) {
          // refresh the stale block summaries of this (class, percent)
          for (uint32_t j = 0; j < NBLK; ++j) {
            if ((sm.valid[ci][j >> 5] >> (j & 31)) & 1u) continue;
            int64_t v[REPLAY_NPT][MAXL];
            uint32_t keys[REPLAY_NPT];
            node_terms(j * REPLAY_BLOCK, v, keys);
            block_scan<MAXL>(sm, v, keys, false, true);   // in-block prefixes; sm.carry = block total
#pragma unroll
            for (int d = 0; d < MAXL; ++d) {
              int64_t mx = max(max(v[0][d], v[1][d]), max(v[2][d], v[3][d]));
#pragma unroll
              for (int o = 16; o; o >>= 1) mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
              if (lane == 0) sm.wmax[wid][d] = mx;
            }
            __syncthreads();
            if (tid < MAXL) {
              int64_t mx = sm.wmax[0][tid];
              for (int w = 1; w < REPLAY_WARPS; ++w) mx = max(mx, sm.wmax[w][tid]);
              const size_t at = ((size_t)ci * NBLK + j) * MAXL + tid;
              a.blk_max[at] = mx;
              a.blk_sum[at] = sm.carry[tid];
            }
            if (tid == 0) {
              a.blk_keys[(size_t)ci * NBLK + j] = sm.carry_keys;
              sm.valid[ci][j >> 5] |= 1u << (j & 31);
            }
            __syncthreads();
          }
          // carry in front of each block: exclusive scan of the block totals, four blocks per thread
          int64_t own[REPLAY_NPT][MAXL], ex[REPLAY_NPT][MAXL];
          uint32_t own_keys[REPLAY_NPT], ex_keys[REPLAY_NPT];
#pragma unroll
          for (int k = 0; k < REPLAY_NPT; ++k) {
            const uint32_t j = REPLAY_NPT * tid + k;
#pragma unroll
            for (int d = 0; d < MAXL; ++d) own[k][d] = j < NBLK ? a.blk_sum[((size_t)ci * NBLK + j) * MAXL + d] : 0;
            own_keys[k] = j < NBLK ? a.blk_keys[(size_t)ci * NBLK + j] : 0u;
          }
          {
            int64_t v[REPLAY_NPT][MAXL];
            uint32_t keys[REPLAY_NPT];
#pragma unroll
            for (int k = 0; k < REPLAY_NPT; ++k) {
              keys[k] = own_keys[k];
#pragma unroll
              for (int d = 0; d < MAXL; ++d) v[k][d] = own[k][d];
            }
            block_scan<MAXL>(sm, v, keys, false, false);
            // keys in front of item k: inclusive keys of item k-1 (of the lane below for k = 0)
            const uint32_t up = __shfl_up_sync(0xffffffffu, keys[REPLAY_NPT - 1], 1);
            const uint32_t front0 = (lane ? up : 0u) | sm.wkeys[wid];
#pragma unroll
            for (int k = 0; k < REPLAY_NPT; ++k) {
              ex_keys[k] = k == 0 ? front0 : keys[k - 1];
#pragma unroll
              for (int d = 0; d < MAXL; ++d) ex[k][d] = v[k][d] - own[k][d];
            }
          }
          // can a prefix inside the block satisfy the need at all?
#pragma unroll
          for (int k = 0; k < REPLAY_NPT; ++k) {
            const uint32_t j = REPLAY_NPT * tid + k;
            if (j >= NBLK) continue;
            bool possible = j > 0 || b0_cached;   // a stale block 0 was just scanned exactly
            if (possible) {
              const uint32_t reach = ex_keys[k] | own_keys[k];
#pragma unroll
              for (int d = 0; d < MAXL; ++d) {
                if ((uint32_t)d >= L) continue;
                const int64_t top = ex[k][d] + a.blk_max[((size_t)ci * NBLK + j) * MAXL + d];
                const int64_t nd = sm.need[d];
                if (d < 4) possible &= top >= nd;
                else if (((need_keys >> d) & 1u) && nd > 0) possible &= ((reach >> d) & 1u) && top >= nd;
              }
            }
            sm.cand[j] = possible ? 1 : 0;
          }
          __syncthreads();
          for (uint32_t j = 0; j < NBLK && !enough; ++j) {
            if (!sm.cand[j]) continue;
            if (tid == j / REPLAY_NPT) {
#pragma unroll
              for (int k = 0; k < REPLAY_NPT; ++k)
                if ((int)(j % REPLAY_NPT) == k) {
#pragma unroll
                  for (int d = 0; d < MAXL; ++d) sm.carry[d] = ex[k][d];
                  sm.carry_keys = ex_keys[k];
                }
            }
            __syncthreads();
            enough = exact_block(j * REPLAY_BLOCK, true, false);
          }
        }
      }
      if (!enough) {                                                 // :141-146, :162-165
        code = BS_PF_ERR_NOT_ENOUGH;
        if (tid == 0) a.gflags[g] |= BS_GROUP_DENIED;                // AddToDenyCache :423-425
      }
    } while (0);
    if (sm.panic) break;   // uniform: written before a barrier every thread has passed

    int32_t chosen = -1;
    uint8_t rdy = 0;
    if (code == BS_PF_PASS) {
      // ---- node choice among the nodes where the pod fits (A5 at percent 1.0): the first in list order, or
      // (SCORED) the best-scoring ----
      const uint32_t rc = cur.rc;   // the pod's own (selector, tolerations) class
      const uint64_t sel = a.rsel[rc], tol = a.rtol[rc];
      int64_t best_s = INT64_MIN;   // SCORED: this thread's best (score, node) so far; node -1 = none
      int32_t best_n = -1;
      for (uint32_t base = lo; base < N; base += REPLAY_BLOCK) {
        int64_t v[REPLAY_NPT][MAXL];
        uint32_t keys[REPLAY_NPT], vis, tok, cf;
        load_quad(base, 0, rc, sel, tol, v, keys, vis, tok, cf);
        const uint32_t usable = vis & tok;
        uint32_t fit = 0, dead = 0;
#pragma unroll
        for (int k = 0; k < REPLAY_NPT; ++k) {
          const bool d0 = !((usable >> k) & 1u) | (v[k][LANE_CPU] < sm.min_req[LANE_CPU]) | (v[k][LANE_MEM] < sm.min_req[LANE_MEM]) |
                          (v[k][LANE_EPH] < sm.min_req[LANE_EPH]) | (v[k][LANE_PODS] < sm.min_req[LANE_PODS]);
          if (d0) dead |= 1u << k;
          if (((usable & cf) >> k) & 1u)
            if (compare_lanes<MAXL>(v[k], keys[k], req, req_keys)) fit |= 1u << k;
        }
        if constexpr (SCORED) {
          // nodes come in ascending order per thread: only a strictly higher score replaces the best
          const int64_t pnz0 = s_pod_nz[par][0], pnz1 = s_pod_nz[par][1];
          [[maybe_unused]] const uint8_t* lrow = nullptr;   // LOC: the pod's IL row (null: IL = 0) and controller bit
          [[maybe_unused]] uint64_t lmask = 0;
          if constexpr (LOC) {
            const uint32_t c = a.w_img ? a.loc_class[cur.p] : 0xffffffffu;   // BS_IMAGE_NONE
            if (c != 0xffffffffu) lrow = a.il + (size_t)c * Npad;
            const uint32_t b = a.w_avoid ? a.avoid_bit[cur.p] : 0xffu;       // BS_AVOID_NONE
            if (b != 0xffu) lmask = 1ull << b;
          }
#pragma unroll
          for (int k = 0; k < REPLAY_NPT; ++k) {
            if (!((fit >> k) & 1u)) continue;
            const uint32_t n = base + REPLAY_NPT * tid + k;
            const int64_t r_cpu = a.nz_live[n] + pnz0, r_mem = a.nz_live[(size_t)Npad + n] + pnz1;
            const int64_t c_cpu = a.nt.alloc[n], c_mem = a.nt.alloc[(size_t)Npad + n];
            int64_t s = pair_score(r_cpu, c_cpu, r_mem, c_mem, a.w);
            if constexpr (RATIO) {
              // lanes >= 2: the live requested and key mask (assume grows them) plus the pod's request, which
              // sm.req already holds as 0 for a key the pod lacks
              uint32_t num = a.ratio.num0, den = a.ratio.den0;
              const uint32_t ap = a.nt.alloc_present[n], rp = a.req_present[n];
#pragma unroll
              for (int d = 0; d < MAXL; ++d) {
                const uint32_t wd = a.ratio.lane_w[d];
                if (!wd) continue;   // uniform; lanes 3 and >= L weigh 0
                int64_t r, c;
                if (d == LANE_CPU) { r = r_cpu; c = c_cpu; }
                else if (d == LANE_MEM) { r = r_mem; c = c_mem; }
                else {
                  c = (d < 4 || ((ap >> d) & 1u)) ? a.nt.alloc[(size_t)d * Npad + n] : 0;
                  const int64_t rn = (d < 4 || ((rp >> d) & 1u)) ? a.requested[(size_t)d * Npad + n] : 0;
                  r = (int64_t)((uint64_t)rn + (uint64_t)req[d]);
                }
                ratio_accumulate(ratio_lane_score(s_tab, r, c), wd, num, den);
              }
              s = (int64_t)((uint64_t)s + (uint64_t)a.ratio.weight * (uint64_t)ratio_round(num, den));
            }
            if constexpr (LOC) {
              const uint64_t il = lrow ? lrow[n] : 0u;
              const uint64_t nav = a.w_avoid ? a.avoid_mask[n] : 0ull;
              s = (int64_t)((uint64_t)s + (uint64_t)a.w_img * il + (uint64_t)a.w_avoid * ((nav & lmask) ? 0u : 100u));
            }
            if (best_n < 0 || s > best_s) { best_s = s; best_n = (int32_t)n; }
          }
        } else {
          if (__syncthreads_or(fit ? 1 : 0)) {
            const uint32_t b = __ballot_sync(0xffffffffu, fit != 0);
            if (b && lane == (uint32_t)(__ffs(b) - 1))
              atomicMin(&sm.first[par], (int32_t)(base + REPLAY_NPT * tid + (uint32_t)(__ffs(fit) - 1)));
            __syncthreads();
            chosen = sm.first[par];
            break;
          }
        }
        if (monotone && base == lo) {
          if (__syncthreads_and(dead == (1u << REPLAY_NPT) - 1u ? 1 : 0)) lo = base + REPLAY_BLOCK;
        }
      }
      if constexpr (SCORED) {
        // the block's best: score descending, then node ascending (node -1 ranks last)
        __shared__ int64_t s_best_s[REPLAY_WARPS];
        __shared__ int32_t s_best_n[REPLAY_WARPS];
        auto better = [](int64_t s, int32_t n, int64_t s2, int32_t n2) {
          return n2 >= 0 && (n < 0 || s2 > s || (s2 == s && n2 < n));
        };
#pragma unroll
        for (int o = 16; o; o >>= 1) {
          const int64_t s2 = __shfl_xor_sync(0xffffffffu, best_s, o);
          const int32_t n2 = __shfl_xor_sync(0xffffffffu, best_n, o);
          if (better(best_s, best_n, s2, n2)) { best_s = s2; best_n = n2; }
        }
        if (lane == 0) { s_best_s[wid] = best_s; s_best_n[wid] = best_n; }
        __syncthreads();
        best_s = s_best_s[0];
        best_n = s_best_n[0];
#pragma unroll
        for (int w = 1; w < REPLAY_WARPS; ++w)
          if (better(best_s, best_n, s_best_s[w], s_best_n[w])) { best_s = s_best_s[w]; best_n = s_best_n[w]; }
        chosen = best_n;   // uniform; the slots are rewritten only after the barrier that ends this step
      }
      if (chosen >= 0) {
        // assume: NodeInfo.AddPod adds the pod's request to `requested` (pods lane: the pod list
        // grows); the node's residual rows follow
        const uint32_t n = (uint32_t)chosen;
        if (tid < L) {
          const uint32_t d = tid;
          int64_t rq = a.requested[(size_t)d * Npad + n];
          if (d != LANE_PODS && (d < 4 || ((req_keys >> d) & 1u))) {
            rq += req[d];
            a.requested[(size_t)d * Npad + n] = rq;
          }
          int64_t sub = rq;
          if (d == LANE_PODS) {
            const int32_t pc = a.pod_count[n] + 1;
            a.pod_count[n] = pc;
            if (rq == 0) sub = pc;                                   // :650-653
          }
          const uint32_t keys_now = a.nt.alloc_present[n] & (a.req_present[n] | req_keys) & ~0xFu;
          const bool present = d < 4 || ((keys_now >> d) & 1u);
          const int64_t cap = a.nt.alloc[(size_t)d * Npad + n];
          a.left[0][(size_t)d * Npad + n] = present ? scale_f32(cap, 1.0f) - sub : 0;
          a.left[1][(size_t)d * Npad + n] = present ? scale_f32(cap, 0.7f) - sub : 0;
        }
        if (tid >= 32 && tid < 32 + 2u * REPLAY_MAX_CLASSES)   // the node's block summaries are stale for every class
          sm.valid[tid - 32][(n / REPLAY_BLOCK) >> 5] &= ~(1u << ((n / REPLAY_BLOCK) & 31));
        if (tid == 32) {
          // NodeInfo.AddPod adds the request's keys of lanes 4..L-1 only: a table has no lane >= L
          const uint32_t rp = a.req_present[n] | (req_keys & ((1u << L) - 1u));
          a.req_present[n] = rp;
          a.both[n] = a.nt.alloc_present[n] & rp & ~0xFu;
        }
        if constexpr (SCORED)   // NodeInfo.AddPod grows the node's non-zero requests by the pod's
          if (tid >= 96 && tid < 98) a.nz_live[(size_t)(tid - 96) * Npad + n] += s_pod_nz[par][tid - 96];
        if (tid == 0) {
          // ---- Permit (core.go:268-309) ----
          if (g < 0 || (uint32_t)g >= G) {
            rdy = 1;
          } else {
            const uint32_t cnt = a.matched[g] + 1;                   // :290 MatchedPodNodes.Set
            a.matched[g] = cnt;
            if (cnt >= (uint32_t)(a.min_member[g] - a.scheduled[g])) {   // :303 uint32
              a.gflags[g] |= BS_GROUP_SCHEDULED;                     // :305
              rdy = 1;
            }
          }
        }
      }
    }
    if (tid == 0) { a.prefilter[qi] = code; a.node[qi] = chosen; a.ready[qi] = rdy; }
    __syncthreads();
    if (chosen >= 0 && g >= 0 && (uint32_t)g < G) {
      if (wid == REPLAY_WARPS - 1) bucket_compute((uint32_t)g / S);
      max_dirty = true;
    }
  }
  if (tid == 0) { a.status[0] = sm.panic; a.status[1] = (int32_t)lo; a.status[2] = sm.monotone; }
}

}  // namespace bsk
