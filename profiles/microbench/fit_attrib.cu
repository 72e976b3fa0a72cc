// fit_attrib.cu — times gang_fit_kernel alone at the bench shape (100000 pods x 10000 nodes, LW=0 LN=3 LS=2:
// the cfg4 lane layout) on synthetic inputs, through the engine's own launcher (fit_inst.cu: tail split
// included), with CUDA events.  Used to attribute the score-mode kernel's time between its arithmetic and its
// store path: build it against copies of csrc/ in which fit.cuh is edited (bulk-store issue compiled out, or the
// arithmetic replaced by a constant score) and run the builds alternately.
//
// build (from the repository root; CSRC = batch-scheduler_b200/csrc or an edited copy of it):
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -I$CSRC -DBS_FIT_SLICE=3 \
//        -o profiles/microbench/fit_attrib profiles/microbench/fit_attrib.cu $CSRC/fit_inst.cu
// run:   ./fit_attrib <label> [iters] [beside] [alloc] [inputs]   prints one JSON line per output mode (score+bitmap,
//        bitmap, none) and per control (ctl-zero, ctl-random: store_pattern2.cu's 4 KB bulk-store pattern writing zeros
//        or random 64-bit words into the score allocation, at the fit kernel's shared memory);
//        beside `sort` / `sort-maxshared`: each launch starts beside `occupier`, which holds the lean queue sort's
//        share of every SM, with the driver's shared-memory carveout or the largest one; `-`: alone;
//        alloc `plain`: the score matrix and fit bitmap come from cudaMalloc; `compressible`: from devmem.hpp, as the
//        engine allocates them; `ab`: both, alternated three times;
//        inputs `r20`: narrow residuals below 2^20 (the default); `r26`: narrow residuals up to 2^26, so fitting
//        scores carry random low words: the least compressible case a narrow shape produces
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "devmem.hpp"
#include "fit.cuh"
#define STORE_PATTERN2_KERNELS_ONLY
#include "store_pattern2.cu"

#define CK(x)                                                                              \
  do {                                                                                     \
    cudaError_t e_ = (x);                                                                  \
    if (e_ != cudaSuccess) {                                                               \
      fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_));   \
      exit(1);                                                                             \
    }                                                                                      \
  } while (0)

// Stand-in for the lean queue sort the engine runs beside the fit kernel: one 256-thread CTA per SM with the sort's
// register (32) and static shared-memory (~13 KB) footprint, resident for `ns` nanoseconds, issuing almost nothing.
__global__ void __launch_bounds__(256, 8) occupier(uint64_t ns, int* sink) {
  __shared__ int pad[13 * 1024 / 4];
  uint32_t v[24];   // live across the wait: the allocation reaches the sort's 32 registers
#pragma unroll
  for (int i = 0; i < 24; ++i) v[i] = threadIdx.x * (i + 3);
  uint64_t t0, t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
  do {
    __nanosleep(20000);
#pragma unroll
    for (int i = 0; i < 24; ++i) asm volatile("add.u32 %0, %0, 1;" : "+r"(v[i]));
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  } while (t - t0 < ns);
  uint32_t x = 0;
#pragma unroll
  for (int i = 0; i < 24; ++i) x ^= v[i];
  pad[threadIdx.x] = (int)(t ^ x);
  __syncthreads();
  if (pad[(threadIdx.x + 1) & 255] == 12345) *sink = 1;
}

static uint64_t rng = 0x9e3779b97f4a7c15ull;
static uint32_t rnd() {
  rng ^= rng << 13; rng ^= rng >> 7; rng ^= rng << 17;
  return (uint32_t)(rng >> 11);
}

int main(int argc, char** argv) {
  const char* label = argc > 1 ? argv[1] : "fit";
  const int iters = argc > 2 ? atoi(argv[2]) : 30;
  const bool with_sort = argc > 3 && !strncmp(argv[3], "sort", 4);
  // "sort": the occupier leaves the shared-memory carveout to the driver; "sort-maxshared": it asks for the largest
  const int carveout = argc > 3 && !strcmp(argv[3], "sort-maxshared") ? (int)cudaSharedmemCarveoutMaxShared : (int)cudaSharedmemCarveoutDefault;
  const char* alloc_arg = argc > 4 ? argv[4] : "plain";
  const bool r26 = argc > 5 && !strcmp(argv[5], "r26");
  constexpr uint32_t LW = 0, LN = 3, LS = 2, L = LW + LN + LS;
  const uint32_t P = 100000, N = 10000;
  const uint32_t Npad = (N + bsk::NODE_TILE - 1) / bsk::NODE_TILE * bsk::NODE_TILE, n_tiles = Npad / bsk::NODE_TILE;
  const uint32_t units = (P + bsk::PODS_PER_CTA - 1) / bsk::PODS_PER_CTA, Prows = units * bsk::PODS_PER_CTA;
  const uint32_t score_pitch = (N + 1) & ~1u, W = (N + 31) / 32, bitmap_pitch = (W + 31) & ~31u;

  // narrow lanes in [0, 2^20) against requests in [0, 2^19) (r26: [0, 2^26) against [0, 2^25), the same fit rate);
  // scaled lanes in units of 2^20; one fit class
  const uint32_t left_mask = r26 ? 0x3ffffff : 0xfffff, req_mask = left_mask >> 1;
  std::vector<int32_t> left_n((size_t)(LN + LS) * Npad, 0);
  for (uint32_t d = 0; d < LN + LS; ++d)
    for (uint32_t n = 0; n < N; ++n) left_n[(size_t)d * Npad + n] = d < LN ? (int32_t)(rnd() & left_mask) : (int32_t)(rnd() % 1000);
  std::vector<int64_t> req((size_t)L * P);
  for (uint32_t d = 0; d < L; ++d)
    for (uint32_t p = 0; p < P; ++p) req[(size_t)d * P + p] = d < LN ? (rnd() & req_mask) : (int64_t)(rnd() % 500) << 20;
  std::vector<bsk::ColBits> cls((size_t)n_tiles * 32);
  for (auto& c : cls) c = (bsk::ColBits)(rnd() | rnd());

  bsk::FitArgs a;
  memset(&a, 0, sizeof(a));
  for (uint32_t k = 0; k < LN; ++k) a.lm.narrow[k] = (uint8_t)k;
  for (uint32_t k = 0; k < LS; ++k) {
    a.lm.scaled[k] = (uint8_t)(LN + k);
    a.lm.sunit[k] = 20;
    a.lm.sshift[k] = 20;
    a.lm.sclamp[k] = 1u << (bsk::FIT_CAP_LOG2 - 20);
  }
  a.lm.LW = LW; a.lm.LN = LN; a.lm.LS = LS;
  int32_t* d_left_n; int64_t* d_req; uint32_t *d_pres, *d_fclass, *d_cnt; bsk::ColBits* d_cls;
  int32_t* d_bn; int64_t* d_bs; unsigned long long* d_packed;
  CK(cudaMalloc(&d_left_n, left_n.size() * 4));
  CK(cudaMalloc(&d_req, req.size() * 8));
  CK(cudaMalloc(&d_cls, cls.size() * sizeof(bsk::ColBits)));
  CK(cudaMalloc(&d_pres, P * 4));
  CK(cudaMalloc(&d_fclass, P * 4));
  CK(cudaMalloc(&d_cnt, Prows * 4));
  CK(cudaMalloc(&d_bn, Prows * 4));
  CK(cudaMalloc(&d_bs, Prows * 8));
  CK(cudaMalloc(&d_packed, Prows * 8));
  // one score matrix and fit bitmap per allocation kind
  const size_t score_bytes = (size_t)Prows * score_pitch * 8, bitmap_bytes = (size_t)Prows * bitmap_pitch * 4;
  struct Alloc { const char* name; bool compressed; int64_t* score; uint32_t* bitmap; };
  std::vector<Alloc> allocs;
  const int attr = bsk::compmem_supported();
  if (strcmp(alloc_arg, "compressible")) {
    Alloc pl{"plain", false, nullptr, nullptr};
    CK(cudaMalloc(&pl.score, score_bytes));
    CK(cudaMalloc(&pl.bitmap, bitmap_bytes));
    allocs.push_back(pl);
  }
  if (strcmp(alloc_arg, "plain")) {
    bsk::CompMem ms, mb;
    const bool gs = bsk::compmem_alloc(&ms, score_bytes), gb = bsk::compmem_alloc(&mb, bitmap_bytes);
    printf("{\"compression_attribute\": %d, \"score_granted\": %s, \"score_bytes\": %zu, \"bitmap_granted\": %s, \"bitmap_bytes\": %zu}\n",
           attr, gs ? "true" : "false", ms.bytes, gb ? "true" : "false", mb.bytes);
    if (!gs || !gb) return 2;
    allocs.push_back({"compressible", true, (int64_t*)ms.p, (uint32_t*)mb.p});
  }
  CK(cudaMemcpy(d_left_n, left_n.data(), left_n.size() * 4, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(d_req, req.data(), req.size() * 8, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(d_cls, cls.data(), cls.size() * sizeof(bsk::ColBits), cudaMemcpyHostToDevice));
  CK(cudaMemset(d_pres, 0xff, P * 4));
  CK(cudaMemset(d_fclass, 0, P * 4));
  a.left_w = nullptr;
  a.left_n = d_left_n;
  a.classfit = d_cls;
  a.req = d_req;
  a.req_present = d_pres;
  a.fit_class = d_fclass;
  a.feasible_count = d_cnt;
  a.best_node = d_bn;
  a.best_score = d_bs;
  a.best_packed = d_packed;
  a.left_w_pitch = (uint64_t)Npad * 8;
  a.left_n_pitch = (uint64_t)Npad * 4;
  a.score_pitch = score_pitch;
  a.bitmap_pitch = bitmap_pitch;
  a.P = P; a.N = N; a.Npad = Npad; a.W = W;

  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, 0));
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  cudaStream_t s_fit, s_sort;
  CK(cudaStreamCreateWithFlags(&s_fit, cudaStreamNonBlocking));
  CK(cudaStreamCreateWithFlags(&s_sort, cudaStreamNonBlocking));
  int* d_sink;
  CK(cudaMalloc(&d_sink, 4));
  struct Mode { const char* name; int out; bool bitmap; };
  const Mode modes[] = {{"score+bitmap", bsk::FIT_OUT_SCORE, true}, {"bitmap", bsk::FIT_OUT_BITMAP, true}, {"none", bsk::FIT_OUT_NONE, false},
                        {"ctl-zero", -1, false}, {"ctl-random", -2, false}};
  // the controls run store_pattern2's 4 KB-segment shape padded to the score-mode fit kernel's shared memory (cfg4)
  constexpr size_t FIT_SMEM = 90880;
  CK(cudaFuncSetAttribute(tma<1, 512, 2, 8, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FIT_SMEM));
  CK(cudaFuncSetAttribute(tma<1, 512, 2, 8, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FIT_SMEM));
  const int reps = allocs.size() > 1 ? 3 : 1;
  for (int rep = 0; rep < reps; ++rep)
  for (const Alloc& al : allocs)
  for (const Mode& m : modes) {
    bsk::FitFn fn = m.out >= 0 ? bsk::fit_lookup_slice3(LW, LN, LS, m.out) : nullptr;
    if (m.out >= 0 && !fn) { fprintf(stderr, "no variant\n"); return 1; }
    bsk::FitArgs b = a;
    b.score = m.out == bsk::FIT_OUT_SCORE ? al.score : nullptr;
    b.fit_bitmap = m.bitmap ? al.bitmap : nullptr;
    auto launch = [&](cudaEvent_t t0, cudaEvent_t t1) -> cudaError_t {
      if (fn) return fn(b, units, s_fit, nullptr, t0, t1);
      if (t0) CK(cudaEventRecord(t0, s_fit));
      if (m.out == -1) tma<1, 512, 2, 8, 1><<<(P + 7) / 8, 256, FIT_SMEM, s_fit>>>((long long*)al.score, (int)P, (int)N);
      else tma<1, 512, 2, 8, 2><<<(P + 7) / 8, 256, FIT_SMEM, s_fit>>>((long long*)al.score, (int)P, (int)N);
      CK(cudaGetLastError());
      return t1 ? cudaEventRecord(t1, s_fit) : cudaSuccess;
    };
    for (int i = 0; i < 3; ++i) CK(launch(nullptr, nullptr));
    CK(cudaDeviceSynchronize());
    std::vector<float> ms(iters);
    for (int i = 0; i < iters; ++i) {
      if (with_sort) {
        CK(cudaDeviceSynchronize());
        CK(cudaFuncSetAttribute(occupier, cudaFuncAttributePreferredSharedMemoryCarveout, carveout));
        occupier<<<prop.multiProcessorCount, 256, 0, s_sort>>>(2400000ull, d_sink);
        CK(cudaGetLastError());
      }
      CK(launch(e0, e1));
      CK(cudaEventSynchronize(e1));
      CK(cudaEventElapsedTime(&ms[i], e0, e1));
    }
    std::vector<float> s = ms;
    std::sort(s.begin(), s.end());
    double mean = 0;
    for (float v : ms) mean += v;
    mean /= iters;
    // checksum of the per-pod results (the score matrix itself is compared by the tests, not here)
    std::vector<uint32_t> cnt(P);
    CK(cudaMemcpy(cnt.data(), d_cnt, P * 4, cudaMemcpyDeviceToHost));
    unsigned long long sum = 0;
    for (uint32_t v : cnt) sum += v;
    printf("{\"build\": \"%s\", \"beside\": \"%s\", \"alloc\": \"%s\", \"inputs\": \"%s\", \"rep\": %d, \"mode\": \"%s\", \"gpu\": \"%s\", "
           "\"iters\": %d, \"median_ms\": %.4f, \"mean_ms\": %.4f, \"min_ms\": %.4f, \"max_ms\": %.4f, \"feasible_sum\": %llu}\n",
           label, argc > 3 ? argv[3] : "-", al.name, r26 ? "r26" : "r20", rep, m.name, prop.name, iters, s[iters / 2], mean, s[0],
           s[iters - 1], sum);
    fflush(stdout);
  }
  return 0;
}
