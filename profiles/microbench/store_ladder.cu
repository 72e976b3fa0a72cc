// store_ladder.cu — where does the score-mode fit kernel's store stream lose time against the bare store pattern?
// Starts from store_pattern2.cu's tma<1,512,2,8> pattern (each warp stages one 4 KB row segment of a 512-node tile
// in one of two shared-memory slabs and one lane hands it to the TMA engine) and adds the structure of
// gang_fit_kernel<0,3,2,FIT_OUT_SCORE> one rung at a time.  No arithmetic: every rung writes the same 100000 x 10000
// int64 matrix (the node index, or values that compress like the real matrix: `values` below), at the kernel's shared
// memory (90 880 B at cfg4's five int32 lanes, two CTAs per SM) unless a rung says otherwise.
//
//   r0_base        the pattern as measured in store_pattern2 (no L2 hint)
//   r1_hint        + the kernel's L2 evict_first policy on the bulk stores
//   r2_ring        + a ninth (producer) warp and the 2-stage TMA input ring of 512-node tiles (5 int32 lanes, 10 KB a
//                    stage) with full/empty mbarriers: all 8 consumer warps release a stage before it is refilled
//   r3_rows4       + 4 rows per warp in the kernel's order: per tile, one segment of row r for r = 0..3, 2 slabs
//   r4_bitmap      + one 128-byte fit-bitmap line per pod every 2 tiles (st.global, no L2 hint)
//   r5_grid        + the kernel's grid: 3125 units of 32 pods, the last partial wave cut into node-range pieces,
//                    per-pod results written plainly or with atomics (pieces)
// Candidate fixes, each on top of r5:
//   r5_stages3     a third input stage (101 120 B)
//   r5_pair        3 input stages, each pod's two consecutive tiles swept back to back (8 KB of one row at a time)
//   r5_bmbulk      the bitmap lines leave as 128-byte bulk stores under the evict_first policy (+4 KB: two line
//                  buffers, so a line is assembled while the previous one is read by the TMA engine)
//   r2_stages3     r2 with a third input stage (how much of r2's step is ring coupling)
//   r3_fb          r3 with each warp's 4 rows written front to back, one after another (the ring streams the tiles
//                  once per row): as many rows in flight as r2
//   r3_rows2       r3 with 2 rows per warp (16-pod CTAs)
//   r5_bmbulk_fb   r5_bmbulk with the rows front to back (the shipped structure)
// Tile re-reads on r5_bmbulk_fb (the ring streams the warp's tile range once per row, four times per CTA):
//   fb_once        the ring streams the tiles once per CTA: later passes complete their stages without a copy (the
//                  bound on what fewer L2 reads of the residual tiles can give)
//   fb_s3          a third input stage
//   fb_mc2, fb_mc4 four passes, each stage multicast to a cluster of 2 or 4 CTAs that share one tile range: every
//                  rank copies its share of the lane rows into every CTA's stage, and a stage is refilled once the
//                  consumer warps of every CTA in the cluster have released it
//   fb_mc2_s3, fb_mc4_s3   the multicast rungs with a third input stage
//
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -I../../batch-scheduler_b200/csrc \
//             -o store_ladder store_ladder.cu
// run:   ./store_ladder <rounds> <iters> <power limit, W> [first round's number] [alloc] [values] [rungs]
//        one JSON line per rung, allocation and round, rungs alternated.  alloc `plain` (cudaMalloc, the default),
//        `compressible` (csrc/devmem.hpp, as the engine allocates the score matrix) or `ab` (both, in turn);
//        values `index` (the node index, the default), `r20` or `r26` (like the real matrix: a per-(row, node) hash
//        makes 18 % of pairs fit, with scores below 2^20 or 2^26, and INT64_MIN elsewhere); rungs: a comma-separated
//        list of rung names (all by default)
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>
#include <cuda_runtime.h>

#include "devmem.hpp"

namespace {

constexpr int T = 512;                  // nodes per tile
constexpr int NB = 2;                   // staging slabs per warp
constexpr int LANES = 5;                // cfg4: 3 narrow + 2 scaled int32 lanes
constexpr uint32_t STAGE = LANES * T * 4;   // 10 KB
constexpr uint32_t SLAB = T * 8;            // 4 KB
constexpr int PODS_PER_CTA = 32;
constexpr uint32_t P = 100000, N = 10000;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n.reg .pred p;\nWAIT_%=:\nmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n@p bra DONE_%=;\nbra WAIT_%=;\n"
      "DONE_%=:\n}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
// the same copy into the stage at this offset of every CTA of the cluster in `mask`, completing on each one's barrier
__device__ __forceinline__ void g2s_mc(void* dst, const void* src, uint32_t bytes, uint64_t* bar, uint16_t mask) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1], %2, [%3], %4;"
               ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)), "h"(mask) : "memory");
}
// arrive on the barrier at this offset in cluster CTA `rank`
__device__ __forceinline__ void mbar_arrive_remote(uint64_t* bar, uint32_t rank) {
  asm volatile("{\n.reg .b32 ra;\nmapa.shared::cluster.u32 ra, %0, %1;\n"
               "mbarrier.arrive.shared::cluster.b64 _, [ra];\n}" ::"r"(smem_u32(bar)), "r"(rank) : "memory");
}
__device__ __forceinline__ void cluster_sync() { asm volatile("barrier.cluster.arrive;\nbarrier.cluster.wait;" ::: "memory"); }
// what the rungs write at (row, node): the node index (vmode 0), or a stand-in for the score matrix (vmode 1 / 2):
// 18 % of pairs fit with a score below 2^20 / 2^26, the rest hold INT64_MIN
__host__ __device__ __forceinline__ long long cell_value(uint32_t vmode, uint32_t row, uint32_t node) {
  if (vmode == 0) return node;
  uint32_t h = row * 0x9e3779b1u ^ (node + 0x7f4a7c15u) * 0x85ebca6bu;
  h ^= h >> 15; h *= 0x2c1b3c6du; h ^= h >> 12; h *= 0x297a2d39u; h ^= h >> 15;
  return (h >> 22) < 184u ? (long long)(h & (vmode == 1 ? 0xfffffu : 0x3ffffffu)) : (long long)INT64_MIN;
}
__device__ __forceinline__ uint64_t evict_first() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
template <bool HINT>
__device__ __forceinline__ void s2g(void* dst, uint32_t src, uint32_t bytes) {
  if (HINT)
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group.L2::cache_hint [%0], [%1], %2, %3;" ::"l"(dst), "r"(src),
                 "r"(bytes), "l"(evict_first()) : "memory");
  else
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read1() { asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

struct LArgs {
  long long* out;
  uint32_t* bitmap;
  const int32_t* left;   // [LANES][Npad]
  uint32_t* cnt;
  unsigned long long* packed;
  int32_t* best;
  uint32_t Npad, pitch, bitmap_pitch, n_full, tail_split, units, vmode;
};

// shared memory: [STAGES] input stages | requests (640 B) | mbarriers | [2 if BM == 2][32 pods][32] bitmap words,
// 128-byte aligned | [8 warps][NB] slabs
__host__ __device__ constexpr uint32_t front_bytes(int stages, int bm) {
  uint32_t b = stages * STAGE + PODS_PER_CTA * LANES * 4;
  b = (b + 7) & ~7u;
  b += 2 * stages * 8 + (bm == 2 ? 2 : 1) * PODS_PER_CTA * 32 * 4;
  return (b + 127) & ~127u;
}
__host__ __device__ constexpr uint32_t smem_bytes(int stages, int bm) { return front_bytes(stages, bm) + 8 * NB * SLAB; }

// HINT: evict_first on the score stores.  RING: producer warp + input ring.  RPW: rows per warp.  BM: bitmap lines
// (0 none, 1 st.global, 2 bulk).  SPLIT: the kernel's grid with tail pieces and per-pod results.  PAIR: two tiles of
// one pod back to back.  FB: each warp's rows front to back.  MC: CTAs per cluster sharing each stage by multicast.
// ONCE: the ring copies the tiles on the first pass only.
template <bool HINT, bool RING, int RPW, int BM, bool SPLIT, int STAGES, bool PAIR, bool FB = false, int MC = 1,
          bool ONCE = false>
__global__ void __launch_bounds__(288, 2) ladder(LArgs a) {
  static_assert(!PAIR || STAGES >= 3, "a pod's tile pair and the next tile's load need three stages");
  static_assert(!FB || (RING && !PAIR), "front to back: one row per pass over the ring's tiles");
  static_assert((MC == 1 && !ONCE) || (FB && BM == 2 && SPLIT), "multicast and single-copy rungs are r5_bmbulk_fb's");
  constexpr int PASSES = FB ? RPW : 1, ROWS = FB ? 1 : RPW;   // FB: the warp writes its rows one after another
  extern __shared__ __align__(128) unsigned char smem[];
  constexpr uint32_t FRONT = front_bytes(STAGES, BM);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + ((STAGES * STAGE + PODS_PER_CTA * LANES * 4 + 7) & ~7u));
  uint64_t* empty = full + STAGES;
  uint32_t* words_all = reinterpret_cast<uint32_t*>(empty + STAGES);
  const uint32_t tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  uint32_t unit = blockIdx.x, piece = 0, npieces = 1;
  const uint32_t rank = blockIdx.x % MC;
  if (MC > 1) {
    // cluster k: units k*MC .. k*MC+MC-1 over one tile range; in the tail, MC units' piece `piece` (n_full % MC == 0)
    const uint32_t cl = blockIdx.x / MC, full_cl = a.n_full / MC;
    unit = cl * MC + rank;
    if (cl >= full_cl) {
      const uint32_t tl = cl - full_cl;
      unit = a.n_full + tl / a.tail_split * MC + rank;
      piece = tl % a.tail_split;
      npieces = a.tail_split;
    }
  } else if (SPLIT && blockIdx.x >= a.n_full) {
    const uint32_t tl = blockIdx.x - a.n_full;
    unit = a.n_full + tl / a.tail_split;
    piece = tl % a.tail_split;
    npieces = a.tail_split;
  }
  const bool live = unit < a.units;   // false: a cluster's spare rank (units % MC), in the protocol but writing nothing
  const uint32_t row0 = unit * (8 * RPW) + wid * RPW;
  const uint32_t n_tiles = a.Npad / T, n_lines = (n_tiles + 1) / 2;
  const uint32_t tile_lo = min(n_tiles, (n_lines * piece / npieces) * 2);
  const uint32_t tile_hi = min(n_tiles, (n_lines * (piece + 1) / npieces) * 2);
  if (RING) {
    if (tid == 0) {
      for (int s = 0; s < STAGES; ++s) {
        mbar_init(&full[s], 1);
        mbar_init(&empty[s], 8 * MC);
      }
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    if (MC > 1) cluster_sync();   // every CTA's barriers exist before any peer copies or arrives
    else __syncthreads();
    if (wid == 8) {
      if (lane == 0)
        for (uint32_t i = 0; i < PASSES * (tile_hi - tile_lo); ++i) {
          const uint32_t t = tile_lo + i % (tile_hi - tile_lo), st = i % STAGES, use = i / STAGES;
          if (use > 0) mbar_wait(&empty[st], (use - 1) & 1);
          if (ONCE && i >= tile_hi - tile_lo) {
            mbar_arrive(&full[st]);
            continue;
          }
          mbar_expect_tx(&full[st], STAGE);
          for (int d = MC > 1 ? rank : 0; d < LANES; d += MC) {
            if (MC > 1)
              g2s_mc(smem + st * STAGE + d * T * 4, a.left + (size_t)d * a.Npad + (size_t)t * T, T * 4, &full[st],
                     (uint16_t)((1u << MC) - 1));
            else
              g2s(smem + st * STAGE + d * T * 4, a.left + (size_t)d * a.Npad + (size_t)t * T, T * 4, &full[st]);
          }
        }
      return;
    }
  } else if (wid >= 8) {
    return;
  }
  const uint32_t slab0 = smem_u32(smem + FRONT) + wid * NB * SLAB;
  uint32_t* words = words_all + wid * RPW * 32;
  uint32_t stage = 0, phase = 0, sb = 0, nseg = 0, bmbuf = 0;
  constexpr uint32_t STEP = PAIR ? 2 : 1;
  for (int pass = 0; pass < PASSES; ++pass)
  for (uint32_t tile = tile_lo; tile < tile_hi; tile += STEP) {
    const uint32_t nt = min(STEP, tile_hi - tile);
    if (RING) {
      uint32_t s = stage, ph = phase;
      for (uint32_t k = 0; k < nt; ++k) {
        mbar_wait(&full[s], ph);
        if (++s == STAGES) { s = 0; ph ^= 1; }
      }
    }
#pragma unroll
    for (int rr = 0; rr < ROWS; ++rr) {
      const int r = FB ? pass : rr;
      for (uint32_t k = 0; k < nt; ++k) {
        const uint32_t t = tile + k, node_base = t * T;
        const uint32_t slab = slab0 + sb * SLAB;
        if (nseg >= NB) {
          if (lane == 0) bulk_wait_read1();
          __syncwarp();
        }
#pragma unroll 4
        for (int j = 0; j < T / 32; ++j)
          asm volatile("st.shared.u64 [%0], %1;" ::"r"(slab + (j * 32 + lane) * 8), "l"(cell_value(a.vmode, row0 + r, node_base + j * 32 + lane)));
        if (BM && lane < T / 32) words[(BM == 2 ? bmbuf * PODS_PER_CTA * 32 : 0) + r * 32 + (t & 1) * (T / 32) + lane] = 0xffffffffu;
        fence_async_smem();
        __syncwarp();
        if (lane == 0) {
          if (live && node_base < a.pitch)
            s2g<HINT>(a.out + (size_t)(row0 + r) * a.pitch + node_base, slab, min((uint32_t)T, a.pitch - node_base) * 8);
          bulk_commit();
        }
        ++nseg;
        sb ^= 1;
      }
    }
    if (RING) {
      __syncwarp();
      for (uint32_t k = 0; k < nt; ++k) {
        if (lane == 0) {
          if (MC > 1)
            for (uint32_t c = 0; c < MC; ++c) mbar_arrive_remote(&empty[stage], c);
          else
            mbar_arrive(&empty[stage]);
        }
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
    }
    const uint32_t tlast = tile + nt - 1;
    if (BM && ((tlast + 1) % 2 == 0 || tlast + 1 == tile_hi)) {
      const uint32_t line = tlast / 2, valid = (tlast % 2 + 1) * (T / 32);
      __syncwarp();
      if (BM == 1) {
        if (lane < valid)
#pragma unroll
          for (int rr = 0; rr < ROWS; ++rr) {
            const int r = FB ? pass : rr;
            a.bitmap[(size_t)(row0 + r) * a.bitmap_pitch + line * 32 + lane] = words[r * 32 + lane];
          }
      } else {
        // staged lines leave with the next segment's bulk group; the other buffer takes the next line
        fence_async_smem();
        __syncwarp();
        if (lane == 0 && live)
#pragma unroll
          for (int rr = 0; rr < ROWS; ++rr) {
            const int r = FB ? pass : rr;
            s2g<true>(a.bitmap + (size_t)(row0 + r) * a.bitmap_pitch + line * 32,
                      smem_u32(words + bmbuf * PODS_PER_CTA * 32 + r * 32), valid * 4);
          }
        bmbuf ^= 1;
      }
    }
  }
  if (lane == 0) {
    if (BM == 2) bulk_commit();
    bulk_wait_read0();
  }
  if (MC > 1) cluster_sync();   // no CTA leaves while a peer may still arrive on its barriers
  if (SPLIT && lane == 0 && live) {
#pragma unroll
    for (int r = 0; r < RPW; ++r) {
      const uint32_t p = row0 + r;
      if (npieces == 1) {
        a.cnt[p] = tile_hi - tile_lo;
        a.best[p] = (int32_t)p;
      } else {
        atomicAdd(&a.cnt[p], tile_hi - tile_lo);
        atomicMax(&a.packed[p], ((unsigned long long)(piece + 1) << 32) | p);
      }
    }
  }
}

struct Rung {
  const char* name;
  void (*fn)(LArgs);
  bool ring, split;
  int rpw;
  uint32_t smem;
  int mc;
};
template <bool HINT, bool RING, int RPW, int BM, bool SPLIT, int STAGES, bool PAIR, bool FB = false, int MC = 1,
          bool ONCE = false>
Rung rung(const char* name) {
  return {name, ladder<HINT, RING, RPW, BM, SPLIT, STAGES, PAIR, FB, MC, ONCE>, RING, SPLIT, RPW, smem_bytes(STAGES, BM), MC};
}

#define CK(x)                                                                            \
  do {                                                                                   \
    cudaError_t e_ = (x);                                                                \
    if (e_ != cudaSuccess) {                                                             \
      fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_)); \
      exit(1);                                                                           \
    }                                                                                    \
  } while (0)

}  // namespace

int main(int argc, char** argv) {
  const int rounds = argc > 1 ? atoi(argv[1]) : 3;
  const int iters = argc > 2 ? atoi(argv[2]) : 25;
  const char* power = argc > 3 ? argv[3] : "unknown";
  const int round0 = argc > 4 ? atoi(argv[4]) : 0;
  const char* alloc_arg = argc > 5 ? argv[5] : "plain";
  const char* values = argc > 6 ? argv[6] : "index";
  const std::string only = argc > 7 ? std::string(",") + argv[7] + "," : std::string();
  const uint32_t vmode = !strcmp(values, "r20") ? 1 : !strcmp(values, "r26") ? 2 : 0;
  const uint32_t Npad = (N + T - 1) / T * T, pitch = N, bitmap_pitch = ((N + 31) / 32 + 31) & ~31u;
  LArgs a{};
  CK(cudaMalloc(&a.bitmap, (size_t)P * bitmap_pitch * 4));
  CK(cudaMalloc(&a.left, (size_t)LANES * Npad * 4));
  CK(cudaMemset((void*)a.left, 0, (size_t)LANES * Npad * 4));
  CK(cudaMalloc(&a.cnt, P * 4));
  CK(cudaMalloc(&a.packed, P * 8));
  CK(cudaMalloc(&a.best, P * 4));
  a.Npad = Npad;
  a.pitch = pitch;
  a.bitmap_pitch = bitmap_pitch;
  a.vmode = vmode;
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, 0));
  // one score matrix per allocation kind (the fit bitmap stays on cudaMalloc, as in the engine)
  const size_t out_bytes = (size_t)P * pitch * 8;
  struct Alloc { const char* name; long long* out; };
  std::vector<Alloc> allocs;
  if (strcmp(alloc_arg, "compressible")) {
    Alloc pl{"plain", nullptr};
    CK(cudaMalloc(&pl.out, out_bytes));
    allocs.push_back(pl);
  }
  if (strcmp(alloc_arg, "plain")) {
    bsk::CompMem m;
    if (!bsk::compmem_alloc(&m, out_bytes)) {
      fprintf(stderr, "compressible memory not granted\n");
      return 2;
    }
    allocs.push_back({"compressible", (long long*)m.p});
  }

  const std::vector<Rung> all = {
      rung<false, false, 1, 0, false, 2, false>("r0_base"),
      rung<true, false, 1, 0, false, 2, false>("r1_hint"),
      rung<true, true, 1, 0, false, 2, false>("r2_ring"),
      rung<true, true, 4, 0, false, 2, false>("r3_rows4"),
      rung<true, true, 4, 1, false, 2, false>("r4_bitmap"),
      rung<true, true, 4, 1, true, 2, false>("r5_grid"),
      rung<true, true, 4, 1, true, 3, false>("r5_stages3"),
      rung<true, true, 4, 1, true, 3, true>("r5_pair"),
      rung<true, true, 4, 2, true, 2, false>("r5_bmbulk"),
      rung<true, true, 1, 0, false, 3, false>("r2_stages3"),
      rung<true, true, 4, 0, false, 2, false, true>("r3_fb"),
      rung<true, true, 2, 0, false, 2, false>("r3_rows2"),
      rung<true, true, 4, 2, true, 2, false, true>("r5_bmbulk_fb"),
      rung<true, true, 4, 2, true, 2, false, true, 1, true>("fb_once"),
      rung<true, true, 4, 2, true, 3, false, true>("fb_s3"),
      rung<true, true, 4, 2, true, 2, false, true, 2>("fb_mc2"),
      rung<true, true, 4, 2, true, 2, false, true, 4>("fb_mc4"),
      rung<true, true, 4, 2, true, 3, false, true, 2>("fb_mc2_s3"),
      rung<true, true, 4, 2, true, 3, false, true, 4>("fb_mc4_s3"),
  };
  std::vector<Rung> rungs;
  for (const Rung& g : all)
    if (only.empty() || only.find(std::string(",") + g.name + ",") != std::string::npos) rungs.push_back(g);
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  for (int rd = 0; rd < rounds; ++rd) {
    for (const Alloc& al : allocs)
    for (const Rung& g : rungs) {
      // the base rungs pad to the kernel's 90 880 B: slabs and stage area alike
      const uint32_t smem = std::max<uint32_t>(g.smem, smem_bytes(2, 1));
      CK(cudaFuncSetAttribute(g.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      const int threads = g.ring ? 288 : 256;
      cudaLaunchConfig_t cfg = {};
      cudaLaunchAttribute attr[1];
      attr[0].id = cudaLaunchAttributeClusterDimension;
      attr[0].val.clusterDim.x = g.mc;
      attr[0].val.clusterDim.y = 1;
      attr[0].val.clusterDim.z = 1;
      cfg.blockDim = dim3(threads);
      cfg.dynamicSmemBytes = smem;
      cfg.attrs = attr;
      cfg.numAttrs = g.mc > 1 ? 1 : 0;
      int occ = 0;
      uint32_t slots = 0;
      if (g.mc > 1) {
        int clusters = 0;
        cfg.gridDim = dim3(g.mc * 1024);
        CK(cudaOccupancyMaxActiveClusters(&clusters, g.fn, &cfg));
        slots = (uint32_t)clusters * g.mc;
        occ = (int)((slots + prop.multiProcessorCount - 1) / prop.multiProcessorCount);
      } else {
        CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, g.fn, threads, smem));
        slots = (uint32_t)occ * prop.multiProcessorCount;
      }
      const uint32_t units = P / (8 * g.rpw);
      LArgs b = a;
      b.out = al.out;
      b.units = units;
      b.n_full = units;
      b.tail_split = 1;
      if (g.split) {
        const uint32_t n_lines = (Npad / T + 1) / 2;
        const uint32_t n_full = units / slots * slots, tail = units - n_full, split = std::min<uint32_t>(8, n_lines);
        if (tail && split > 1 && tail * 10 < slots * 9) {
          b.n_full = n_full;
          b.tail_split = split;
        }
      }
      const uint32_t tail_units = units - b.n_full;
      const uint32_t grid = g.mc > 1 ? b.n_full + (tail_units + g.mc - 1) / g.mc * g.mc * b.tail_split
                                     : b.n_full + tail_units * b.tail_split;
      cfg.gridDim = dim3(grid);
      auto launch = [&] {
        if (g.split && b.tail_split > 1) {
          const uint32_t p0 = b.n_full * PODS_PER_CTA;
          CK(cudaMemsetAsync(b.cnt + p0, 0, (size_t)(P - p0) * 4));
          CK(cudaMemsetAsync(b.packed + p0, 0, (size_t)(P - p0) * 8));
        }
        CK(cudaEventRecord(e0));
        CK(cudaLaunchKernelEx(&cfg, g.fn, b));
        CK(cudaEventRecord(e1));
        CK(cudaEventSynchronize(e1));
      };
      CK(cudaMemset(b.out, 0xff, out_bytes));
      for (int i = 0; i < 3; ++i) launch();
      std::vector<float> ms(iters);
      for (int i = 0; i < iters; ++i) {
        launch();
        CK(cudaEventElapsedTime(&ms[i], e0, e1));
      }
      CK(cudaGetLastError());
      std::sort(ms.begin(), ms.end());
      // check the first, a middle and the last row at both ends and inside
      bool ok = true;
      for (uint32_t row : {0u, P / 2 + 7, P - 1})
        for (uint32_t n : {0u, 511u, 4100u, N - 1}) {
          long long v;
          CK(cudaMemcpy(&v, b.out + (size_t)row * pitch + n, 8, cudaMemcpyDeviceToHost));
          ok = ok && v == cell_value(vmode, row, n);
        }
      printf("{\"rung\": \"%s\", \"alloc\": \"%s\", \"values\": \"%s\", \"round\": %d, \"median_ms\": %.4f, \"min_ms\": %.4f, "
             "\"iters\": %d, \"grid\": %u, \"cluster\": %d, \"threads\": %d, \"smem\": %u, \"ctas_per_sm\": %d, \"ok\": %s, "
             "\"gpu\": \"%s\", \"power_limit_w\": \"%s\"}\n",
             g.name, al.name, values, round0 + rd, ms[iters / 2], ms[0], iters, grid, g.mc, threads, smem, occ,
             ok ? "true" : "false", prop.name, power);
      fflush(stdout);
    }
  }
  return 0;
}
