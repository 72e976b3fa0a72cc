// store_pattern.cu — what bounds a write-only P x N int64 matrix kernel on H100?
// Every variant writes the same 100000 x 10000 x 8 B = 8.0 GB with 8-byte streaming stores:
//   fill      : flat grid-stride fill (cudaMemset-like reference)
//   rows32    : the gang_fit pattern — CTA owns 32 rows, 8 warps x 4 rows, sweeps 512-node tiles,
//               per tile each warp writes 16 x 256 B per row, rows interleaved
//   rows32_po : same ownership, pods-outer: a warp finishes a row's 4 KB tile segment before the next row
//   cta_row   : CTA owns 32 rows but all 8 warps cooperate on ONE row at a time (2 KB per step)
//   rows8     : CTA owns 8 rows (1 per warp), 4x more CTAs
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o store_pattern store_pattern.cu
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

constexpr int TILE = 512;

__global__ void fill(long long* p, size_t n) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) __stcs(p + i, 7ll);
}
template <int ROWS_PER_WARP, bool PODS_OUTER>
__global__ void rows(long long* out, int P, int N) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int row0 = (blockIdx.x * nw + wid) * ROWS_PER_WARP;
  for (int base = 0; base < N; base += TILE) {
    if (PODS_OUTER) {
      for (int r = 0; r < ROWS_PER_WARP; ++r)
        for (int j = 0; j < TILE / 32; ++j) {
          const int n = base + j * 32 + lane;
          if (row0 + r < P && n < N) __stcs(out + (size_t)(row0 + r) * N + n, (long long)(n + r));
        }
    } else {
      for (int j = 0; j < TILE / 32; ++j)
        for (int r = 0; r < ROWS_PER_WARP; ++r) {
          const int n = base + j * 32 + lane;
          if (row0 + r < P && n < N) __stcs(out + (size_t)(row0 + r) * N + n, (long long)(n + r));
        }
    }
  }
}
__global__ void cta_row(long long* out, int P, int N) {
  const int row0 = blockIdx.x * 32;
  for (int base = 0; base < N; base += TILE)
    for (int r = 0; r < 32; ++r)
      for (int k = threadIdx.x; k < TILE; k += blockDim.x) {
        const int n = base + k;
        if (row0 + r < P && n < N) __stcs(out + (size_t)(row0 + r) * N + n, (long long)(n + r));
      }
}
template <class F>
float timeit(F f) {
  cudaEvent_t a, b;
  cudaEventCreate(&a); cudaEventCreate(&b);
  for (int i = 0; i < 3; ++i) f();
  float best = 1e9f;
  for (int i = 0; i < 10; ++i) {
    cudaEventRecord(a); f(); cudaEventRecord(b); cudaEventSynchronize(b);
    float ms; cudaEventElapsedTime(&ms, a, b); best = ms < best ? ms : best;
  }
  return best;
}
int main() {
  const int P = 100000, N = 10000;
  const size_t n = (size_t)P * N;
  long long* d;
  cudaMalloc(&d, n * 8);
  auto rep = [&](const char* name, float ms) { printf("%-10s %.3f ms  %.0f GB/s\n", name, ms, n * 8 / ms / 1e6); };
  rep("fill", timeit([&] { fill<<<132 * 8, 256>>>(d, n); }));
  rep("rows32", timeit([&] { rows<4, false><<<(P + 31) / 32, 256>>>(d, P, N); }));
  rep("rows32_po", timeit([&] { rows<4, true><<<(P + 31) / 32, 256>>>(d, P, N); }));
  rep("cta_row", timeit([&] { cta_row<<<(P + 31) / 32, 256>>>(d, P, N); }));
  rep("rows8", timeit([&] { rows<1, false><<<(P + 7) / 8, 256>>>(d, P, N); }));
  rep("rows16", timeit([&] { rows<2, false><<<(P + 15) / 16, 256>>>(d, P, N); }));
  cudaError_t e = cudaDeviceSynchronize();
  printf("status: %s\n", cudaGetErrorString(e));
  return 0;
}
