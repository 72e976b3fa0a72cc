// store_ladder.cu — where does the score-mode fit kernel's store stream lose time against the bare store pattern?
// Starts from store_pattern2.cu's tma<1,512,2,8> pattern (each warp stages one 4 KB row segment of a 512-node tile
// in one of two shared-memory slabs and one lane hands it to the TMA engine) and adds the structure of
// gang_fit_kernel<0,3,2,FIT_OUT_SCORE> one rung at a time.  No arithmetic: every rung writes `node index` into the
// same 100000 x 10000 int64 matrix, at the kernel's shared memory (90 880 B at cfg4's five int32 lanes, two CTAs
// per SM) unless a rung says otherwise.
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
//   r5_bmbulk_fb   r5_bmbulk with the rows front to back
//
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o store_ladder store_ladder.cu
// run:   ./store_ladder <rounds> <iters> <power limit, W> [first round's number]   one JSON line per rung and round,
//        rungs alternated
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>
#include <cuda_runtime.h>

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
  uint32_t Npad, pitch, bitmap_pitch, n_full, tail_split;
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
// one pod back to back.
template <bool HINT, bool RING, int RPW, int BM, bool SPLIT, int STAGES, bool PAIR, bool FB = false>
__global__ void __launch_bounds__(288, 2) ladder(LArgs a) {
  static_assert(!PAIR || STAGES >= 3, "a pod's tile pair and the next tile's load need three stages");
  static_assert(!FB || (RING && !PAIR), "front to back: one row per pass over the ring's tiles");
  constexpr int PASSES = FB ? RPW : 1, ROWS = FB ? 1 : RPW;   // FB: the warp writes its rows one after another
  extern __shared__ __align__(128) unsigned char smem[];
  constexpr uint32_t FRONT = front_bytes(STAGES, BM);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + ((STAGES * STAGE + PODS_PER_CTA * LANES * 4 + 7) & ~7u));
  uint64_t* empty = full + STAGES;
  uint32_t* words_all = reinterpret_cast<uint32_t*>(empty + STAGES);
  const uint32_t tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  uint32_t unit = blockIdx.x, piece = 0, npieces = 1;
  if (SPLIT && blockIdx.x >= a.n_full) {
    const uint32_t tl = blockIdx.x - a.n_full;
    unit = a.n_full + tl / a.tail_split;
    piece = tl % a.tail_split;
    npieces = a.tail_split;
  }
  const uint32_t row0 = unit * (8 * RPW) + wid * RPW;
  const uint32_t n_tiles = a.Npad / T, n_lines = (n_tiles + 1) / 2;
  const uint32_t tile_lo = min(n_tiles, (n_lines * piece / npieces) * 2);
  const uint32_t tile_hi = min(n_tiles, (n_lines * (piece + 1) / npieces) * 2);
  if (RING) {
    if (tid == 0) {
      for (int s = 0; s < STAGES; ++s) {
        mbar_init(&full[s], 1);
        mbar_init(&empty[s], 8);
      }
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (wid == 8) {
      if (lane == 0)
        for (uint32_t i = 0; i < PASSES * (tile_hi - tile_lo); ++i) {
          const uint32_t t = tile_lo + i % (tile_hi - tile_lo), st = i % STAGES, use = i / STAGES;
          if (use > 0) mbar_wait(&empty[st], (use - 1) & 1);
          mbar_expect_tx(&full[st], STAGE);
          for (int d = 0; d < LANES; ++d)
            g2s(smem + st * STAGE + d * T * 4, a.left + (size_t)d * a.Npad + (size_t)t * T, T * 4, &full[st]);
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
          asm volatile("st.shared.u64 [%0], %1;" ::"r"(slab + (j * 32 + lane) * 8), "l"((long long)(node_base + j * 32 + lane)));
        if (BM && lane < T / 32) words[(BM == 2 ? bmbuf * PODS_PER_CTA * 32 : 0) + r * 32 + (t & 1) * (T / 32) + lane] = 0xffffffffu;
        fence_async_smem();
        __syncwarp();
        if (lane == 0) {
          if (node_base < a.pitch)
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
        if (lane == 0) mbar_arrive(&empty[stage]);
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
        if (lane == 0)
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
  if (SPLIT && lane == 0) {
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
};
template <bool HINT, bool RING, int RPW, int BM, bool SPLIT, int STAGES, bool PAIR, bool FB = false>
Rung rung(const char* name) {
  return {name, ladder<HINT, RING, RPW, BM, SPLIT, STAGES, PAIR, FB>, RING, SPLIT, RPW, smem_bytes(STAGES, BM)};
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
  const uint32_t Npad = (N + T - 1) / T * T, pitch = N, bitmap_pitch = ((N + 31) / 32 + 31) & ~31u;
  LArgs a{};
  CK(cudaMalloc(&a.out, (size_t)P * pitch * 8));
  CK(cudaMalloc(&a.bitmap, (size_t)P * bitmap_pitch * 4));
  CK(cudaMalloc(&a.left, (size_t)LANES * Npad * 4));
  CK(cudaMemset((void*)a.left, 0, (size_t)LANES * Npad * 4));
  CK(cudaMalloc(&a.cnt, P * 4));
  CK(cudaMalloc(&a.packed, P * 8));
  CK(cudaMalloc(&a.best, P * 4));
  a.Npad = Npad;
  a.pitch = pitch;
  a.bitmap_pitch = bitmap_pitch;
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, 0));

  const std::vector<Rung> rungs = {
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
  };
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  for (int rd = 0; rd < rounds; ++rd) {
    for (const Rung& g : rungs) {
      // the base rungs pad to the kernel's 90 880 B: slabs and stage area alike
      const uint32_t smem = std::max<uint32_t>(g.smem, smem_bytes(2, 1));
      CK(cudaFuncSetAttribute(g.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      const int threads = g.ring ? 288 : 256;
      int occ = 0;
      CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, g.fn, threads, smem));
      const uint32_t units = P / (8 * g.rpw);
      LArgs b = a;
      b.n_full = units;
      b.tail_split = 1;
      if (g.split) {
        const uint32_t slots = (uint32_t)occ * prop.multiProcessorCount, n_lines = (Npad / T + 1) / 2;
        const uint32_t n_full = units / slots * slots, tail = units - n_full, split = std::min<uint32_t>(8, n_lines);
        if (tail && split > 1 && tail * 10 < slots * 9) {
          b.n_full = n_full;
          b.tail_split = split;
        }
      }
      const uint32_t grid = b.n_full + (units - b.n_full) * b.tail_split;
      auto launch = [&] {
        if (g.split && b.tail_split > 1) {
          const uint32_t p0 = b.n_full * PODS_PER_CTA;
          CK(cudaMemsetAsync(b.cnt + p0, 0, (size_t)(P - p0) * 4));
          CK(cudaMemsetAsync(b.packed + p0, 0, (size_t)(P - p0) * 8));
        }
        CK(cudaEventRecord(e0));
        g.fn<<<grid, threads, smem>>>(b);
        CK(cudaEventRecord(e1));
        CK(cudaEventSynchronize(e1));
      };
      CK(cudaMemset(a.out, 0xff, (size_t)P * pitch * 8));
      for (int i = 0; i < 3; ++i) launch();
      std::vector<float> ms(iters);
      for (int i = 0; i < iters; ++i) {
        launch();
        CK(cudaEventElapsedTime(&ms[i], e0, e1));
      }
      CK(cudaGetLastError());
      std::sort(ms.begin(), ms.end());
      // every row holds its node indices: check the first, a middle and the last row at both ends
      bool ok = true;
      for (uint32_t row : {0u, P / 2 + 7, P - 1})
        for (uint32_t n : {0u, 511u, N - 1}) {
          long long v;
          CK(cudaMemcpy(&v, a.out + (size_t)row * pitch + n, 8, cudaMemcpyDeviceToHost));
          ok = ok && v == (long long)n;
        }
      printf("{\"rung\": \"%s\", \"round\": %d, \"median_ms\": %.4f, \"min_ms\": %.4f, \"iters\": %d, \"grid\": %u, "
             "\"threads\": %d, \"smem\": %u, \"ctas_per_sm\": %d, \"ok\": %s, \"gpu\": \"%s\", \"power_limit_w\": \"%s\"}\n",
             g.name, round0 + rd, ms[iters / 2], ms[0], iters, grid, threads, smem, occ, ok ? "true" : "false", prop.name, power);
      fflush(stdout);
    }
  }
  return 0;
}
