// priority_inst.cu — the priority lists' kernels (priority.cuh), compiled once per slice (build.py, -DBS_PRIO_SLICE=k
// for k = 0..5) so that the 96 builds of priority_pod_kernel compile in parallel with the other units: slice k holds
// the 16 builds of lane bound 5, 9 or 16 (k / 2 = 0, 1, 2) with IPA off (even k) or on (odd k), and slice 0 also the
// LOC and IPA pre-passes.  engine.cu reaches the builds through launch_priority_slice and the pre-passes through
// launch_locality_prepass and launch_interpod_prepass.
#define BS_KERNELS_HELPERS_ONLY   // kernels.cuh's round kernels live in engine.cu
#include "priority.cuh"

#ifndef BS_PRIO_SLICE
#error "compile with -DBS_PRIO_SLICE=0..5"
#endif

namespace bsk {

template <int MAXL, uint32_t IPA>
void launch_priority_slice(uint32_t terms, uint32_t grid, const PriorityIpaArgs& a, cudaStream_t s) {
  with_flags<PRIO_IPA>(terms % PRIO_IPA, [&](auto low) {
    constexpr uint32_t T = IPA | decltype(low)::value;
    priority_pod_kernel<MAXL, (T & PRIO_RATIO) != 0, (T & PRIO_PREF) != 0, (T & PRIO_LOC) != 0, (T & PRIO_SPREAD) != 0,
                        (T & PRIO_IPA) != 0><<<grid, PRIO_THREADS, 0, s>>>(a);
  });
}
constexpr int SLICE_MAXL[] = {5, 9, 16};
template void launch_priority_slice<SLICE_MAXL[BS_PRIO_SLICE / 2], BS_PRIO_SLICE % 2 * PRIO_IPA>(
    uint32_t, uint32_t, const PriorityIpaArgs&, cudaStream_t);

#if BS_PRIO_SLICE == 0
namespace {

// The LOC pre-pass.  ImageLocality's per-name score depends on how many snapshot nodes report the name, and its sum
// over a pod's containers only on the pod's image class, so both are built once per (node side, pod side) and the
// scoring sweep reads one byte per pair.
//
// K1f image_spread_kernel — one warp per dictionary name: NumNodes = the popcount of the name's bit row over the
// n_nodes real nodes, then scaled = (int64)((double)size * ((double)NumNodes / (double)n_nodes)).  The explicit
// round-to-nearest intrinsics keep each operation a separate binary64 rounding whatever -fmad says.
__global__ void __launch_bounds__(LOC_THREADS) image_spread_kernel(const uint32_t* bits, const int64_t* size,
                                                                   int64_t* scaled, uint32_t n_images, uint32_t n_nodes,
                                                                   uint32_t words) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t img = (blockIdx.x * LOC_THREADS + threadIdx.x) >> 5;
  if (img >= n_images) return;   // warp-uniform
  const uint32_t* row = bits + (size_t)img * words;
  uint32_t cnt = 0;
  for (uint32_t w = lane; w < words; w += 32) {
    uint32_t x = row[w];
    const uint32_t lo = w * 32;
    if (lo + 32 > n_nodes) x &= (1u << (n_nodes - lo)) - 1u;   // n_nodes - lo < 32: bits past the last node
    cnt += __popc(x);
  }
  cnt = __reduce_add_sync(0xffffffffu, cnt);
  if (lane == 0) {
    const double spread = __ddiv_rn((double)cnt, (double)n_nodes);
    scaled[img] = __double2ll_rz(__dmul_rn((double)size[img], spread));
  }
}

// K1g locality_class_kernel — IL of every (class, node): a thread per node, the class's ids and their scaled sizes in
// shared memory (at most BS_LOC_CLASS_MAX).  Padding nodes get 0.
constexpr int64_t IL_MIN = 23ll << 20, IL_MAX = 1000ll << 20;   // ImageLocality's thresholds, 23 MiB and 1000 MiB
__global__ void __launch_bounds__(LOC_THREADS) locality_class_kernel(const uint32_t* class_offset,
                                                                     const uint32_t* class_images,
                                                                     const uint32_t* bits, const int64_t* scaled,
                                                                     uint8_t* il, uint32_t n_classes, uint32_t n_nodes,
                                                                     uint32_t Npad, uint32_t words) {
  __shared__ uint32_t s_img[64];
  __shared__ int64_t s_scaled[64];
  const uint32_t i = blockIdx.x * LOC_THREADS + threadIdx.x;
  for (uint32_t c = blockIdx.y; c < n_classes; c += gridDim.y) {
    const uint32_t o0 = class_offset[c], n = class_offset[c + 1] - o0;
    __syncthreads();
    if (threadIdx.x < n) {
      const uint32_t id = class_images[o0 + threadIdx.x];
      s_img[threadIdx.x] = id;
      s_scaled[threadIdx.x] = scaled[id];
    }
    __syncthreads();
    if (i >= Npad) continue;
    int64_t sum = 0;
    if (i < n_nodes)
      for (uint32_t k = 0; k < n; ++k)
        if ((bits[(size_t)s_img[k] * words + (i >> 5)] >> (i & 31)) & 1u) sum += s_scaled[k];
    sum = min(max(sum, IL_MIN), IL_MAX);
    il[(size_t)c * Npad + i] = i < n_nodes ? (uint8_t)(100 * (sum - IL_MIN) / (IL_MAX - IL_MIN)) : 0;
  }
}

// The IPA pre-pass.  raw(c, n) = sum over class c's entries (t, own, match) of own * M[t][v] + match * S[t][v], v = n's
// value of key(t), with M / S the sums of match / own over the bound pods whose node has value v (bsched.h): an
// identity, grouped by term.  Integer sums in any order give the same table, so the result is bit-exact.
//
// K1h interpod_mass_kernel — a thread per bound pod, walking its class's entries in step with its warp: entry k of every
// lane at once.  Bound pods of one class on nodes with one value of a key hit one (term, value) slot, so the lanes with
// the same slot add theirs with __match_any_sync and __reduce_add_sync (|own| sum <= 32 x 2^16, no wrap) and one lane
// of each slot does the two int64 atomics.  Every lane of a warp reaches the warp-wide calls: no lane returns early.
__global__ void __launch_bounds__(LOC_THREADS) interpod_mass_kernel(const uint32_t* bound_node,
                                                                    const uint32_t* bound_class, uint32_t n_bound,
                                                                    InterpodClasses cl, const uint32_t* topo,
                                                                    const uint32_t* term_key, const uint32_t* term_off,
                                                                    uint32_t n_nodes, int64_t* ms) {
  const uint32_t e = blockIdx.x * LOC_THREADS + threadIdx.x, lane = threadIdx.x & 31;
  const uint32_t c = e < n_bound ? bound_class[e] : IPA_NONE;
  uint32_t o0 = 0, n = 0, node = 0;
  if (c != IPA_NONE) {
    o0 = cl.offset[c];
    n = cl.offset[c + 1] - o0;
    node = bound_node[e];
  }
  const uint32_t rounds = __reduce_max_sync(0xffffffffu, n);
  for (uint32_t k = 0; k < rounds; ++k) {
    uint64_t slot = ~0ull;
    int32_t own = 0;
    uint32_t match = 0;
    if (k < n) {
      const uint32_t t = cl.term[o0 + k];
      const uint32_t v = topo[(size_t)term_key[t] * n_nodes + node];
      if (v != TOPO_NONE) {
        slot = (uint64_t)term_off[t] + v;
        own = cl.own[o0 + k];
        match = cl.match[o0 + k];
      }
    }
    const uint32_t peers = __match_any_sync(0xffffffffu, slot);
    if (slot != ~0ull) {
      const uint32_t m = __reduce_add_sync(peers, match);
      const int32_t w = (int32_t)__reduce_add_sync(peers, (uint32_t)own);
      if (lane == (uint32_t)(__ffs(peers) - 1)) {
        if (m) atomicAdd((unsigned long long*)&ms[2 * slot], (unsigned long long)m);
        if (w) atomicAdd((unsigned long long*)&ms[2 * slot + 1], (unsigned long long)(int64_t)w);
      }
    }
  }
}

// K1i interpod_class_kernel — raw of every (pod class, node): a thread per node, the class's entries (at most
// BS_IPA_CLASS_MAX) with their keys and slots in shared memory.  Padding nodes get 0.
__global__ void __launch_bounds__(LOC_THREADS) interpod_class_kernel(InterpodClasses cl, const uint32_t* topo,
                                                                     const uint32_t* term_key,
                                                                     const uint32_t* term_off, const int64_t* ms,
                                                                     int64_t* raw, uint32_t n_nodes, uint32_t Npad) {
  __shared__ uint32_t s_key[IPA_CLASS_MAX], s_off[IPA_CLASS_MAX];
  __shared__ int32_t s_own[IPA_CLASS_MAX];
  __shared__ uint8_t s_match[IPA_CLASS_MAX];
  const uint32_t i = blockIdx.x * LOC_THREADS + threadIdx.x;
  for (uint32_t c = blockIdx.y; c < cl.n_classes; c += gridDim.y) {
    const uint32_t o0 = cl.offset[c], n = cl.offset[c + 1] - o0;
    __syncthreads();
    if (threadIdx.x < n) {
      const uint32_t t = cl.term[o0 + threadIdx.x];
      s_key[threadIdx.x] = term_key[t];
      s_off[threadIdx.x] = term_off[t];
      s_own[threadIdx.x] = cl.own[o0 + threadIdx.x];
      s_match[threadIdx.x] = cl.match[o0 + threadIdx.x];
    }
    __syncthreads();
    if (i >= Npad) continue;
    int64_t r = 0;
    if (i < n_nodes)
      for (uint32_t k = 0; k < n; ++k) {
        const uint32_t v = topo[(size_t)s_key[k] * n_nodes + i];
        if (v == TOPO_NONE) continue;
        const longlong2 q = reinterpret_cast<const longlong2*>(ms)[(size_t)s_off[k] + v];
        r += (int64_t)s_own[k] * q.x + (s_match[k] ? q.y : 0);
      }
    raw[(size_t)c * Npad + i] = r;
  }
}

}  // namespace

cudaError_t launch_locality_prepass(const uint32_t* bits, const int64_t* size, int64_t* scaled, uint32_t n_images,
                                    const uint32_t* class_offset, const uint32_t* class_images, uint8_t* il,
                                    uint32_t n_classes, uint32_t n_nodes, uint32_t Npad, cudaStream_t s) {
  const uint32_t words = (n_nodes + 31) / 32;
  if (n_images && n_nodes)
    image_spread_kernel<<<(n_images + LOC_THREADS / 32 - 1) / (LOC_THREADS / 32), LOC_THREADS, 0, s>>>(
        bits, size, scaled, n_images, n_nodes, words);
  const dim3 grid((Npad + LOC_THREADS - 1) / LOC_THREADS, n_classes < 65535u ? n_classes : 65535u);
  locality_class_kernel<<<grid, LOC_THREADS, 0, s>>>(class_offset, class_images, bits, scaled, il, n_classes, n_nodes,
                                                     Npad, words);
  return cudaGetLastError();
}

cudaError_t launch_interpod_prepass(bool mass, const uint32_t* topo, const uint32_t* term_key, const uint32_t* term_off,
                                    const uint32_t* bound_node, const uint32_t* bound_class, uint32_t n_bound,
                                    const InterpodClasses& bound, const InterpodClasses& pods, int64_t* ms,
                                    int64_t* raw, uint32_t n_nodes, uint32_t Npad, cudaStream_t s) {
  if (mass && n_bound)
    interpod_mass_kernel<<<(n_bound + LOC_THREADS - 1) / LOC_THREADS, LOC_THREADS, 0, s>>>(
        bound_node, bound_class, n_bound, bound, topo, term_key, term_off, n_nodes, ms);
  const dim3 grid((Npad + LOC_THREADS - 1) / LOC_THREADS, pods.n_classes < 65535u ? pods.n_classes : 65535u);
  interpod_class_kernel<<<grid, LOC_THREADS, 0, s>>>(pods, topo, term_key, term_off, ms, raw, n_nodes, Npad);
  return cudaGetLastError();
}

#endif

}  // namespace bsk
