// interpod_filter.cuh — the pre-pass of kube-scheduler v1.17's MatchInterPodAffinity filter (include/bsched.h
// bs_set_interpod_filter, DESIGN.md §2).  It runs at the first evaluation after either side changes or the filter is
// switched on, and leaves one pass bit per (filter class, node) for class_fit_kernel and reason_class_kernel, and two
// more bit planes that tell the failing step apart for reason_pod_kernel.  Steady rounds launch nothing here.
//
// Presence is per term and per value of the term's key: slot term_off[t] + v.  Upstream keys its topology-pair maps by
// (key, value) and not by term, but every map test reduces to a per-term one (DESIGN.md §2), so bits per (term, value)
// decide exactly what the maps decide.
#pragma once
#include "common.cuh"

namespace bsk {

constexpr int IPF_THREADS = 256;

// The filter's class tables on the device.  Bound classes: (term, own, match); pod classes: (term, role), self_match.
struct IpfBound {
  const uint32_t* node;    // [n_bound]
  const uint32_t* cls;     // [n_bound] or BS_IPF_NONE
  const uint32_t* offset;  // [classes + 1]
  const uint32_t* term;
  const int32_t* own;      // 0 or 1
  const uint8_t* match;    // 0 or 1
  uint32_t n_bound;
};
struct IpfPods {
  const uint32_t* offset;  // [n_classes + 1]
  const uint32_t* term;
  const uint8_t* role;     // BS_IPF_AFFINITY / ANTI / EXISTING
  const uint8_t* self_match;
  uint32_t n_classes;
};
struct IpfTopo {
  const uint32_t* topo;      // [keys][n_nodes] value or BS_TOPO_NONE
  const uint32_t* term_key;  // [terms]
  const uint32_t* term_off;  // [terms] first slot of the term
  uint32_t n_nodes;
};

// The kernels are defined once, in engine.cu; replay_inst.cu (BS_KERNELS_HELPERS_ONLY) needs the types above only.
#ifndef BS_KERNELS_HELPERS_ONLY
// K1j ipf_presence_kernel — a thread per bound pod, walking its class's entries in step with its warp (entry k of every
// lane at once).  For an entry whose key the pod's node carries (value v): match sets bit term_off + v of the match
// plane and adds one to the term's count, own sets the bit of the own plane.  Lanes that hit one plane word combine
// their bits with __match_any_sync and __reduce_or_sync first, and one lane per word does the atomicOr: a hostname
// key spreads a warp over many words, a zone key puts it on a handful.  The counts combine the same way per term.
// Every lane reaches the warp-wide calls: no lane returns early.
__global__ void __launch_bounds__(IPF_THREADS) ipf_presence_kernel(IpfBound b, IpfTopo tp, uint32_t* mbits,
                                                                    uint32_t* obits, uint32_t* hits) {
  const uint32_t e = blockIdx.x * IPF_THREADS + threadIdx.x, lane = threadIdx.x & 31;
  const uint32_t c = e < b.n_bound ? b.cls[e] : BS_IPF_NONE;
  uint32_t o0 = 0, n = 0, node = 0;
  if (c != BS_IPF_NONE) {
    o0 = b.offset[c];
    n = b.offset[c + 1] - o0;
    node = b.node[e];
  }
  const uint32_t rounds = __reduce_max_sync(0xffffffffu, n);
  for (uint32_t k = 0; k < rounds; ++k) {
    uint64_t mword = ~0ull, oword = ~0ull;
    uint32_t bit = 0, term = BS_IPF_NONE;
    if (k < n) {
      const uint32_t t = b.term[o0 + k];
      const uint32_t v = tp.topo[(size_t)tp.term_key[t] * tp.n_nodes + node];
      if (v != BS_TOPO_NONE) {
        const uint64_t slot = (uint64_t)tp.term_off[t] + v;
        bit = 1u << (slot & 31);
        if (b.match[o0 + k]) {
          mword = slot >> 5;
          term = t;
        }
        if (b.own[o0 + k]) oword = slot >> 5;
      }
    }
    const uint32_t mp = __match_any_sync(0xffffffffu, mword);
    const uint32_t mb = __reduce_or_sync(mp, mword != ~0ull ? bit : 0u);
    if (mword != ~0ull && lane == (uint32_t)(__ffs(mp) - 1)) atomicOr(&mbits[mword], mb);
    const uint32_t op = __match_any_sync(0xffffffffu, oword);
    const uint32_t ob = __reduce_or_sync(op, oword != ~0ull ? bit : 0u);
    if (oword != ~0ull && lane == (uint32_t)(__ffs(op) - 1)) atomicOr(&obits[oword], ob);
    const uint32_t tpeers = __match_any_sync(0xffffffffu, term);
    if (term != BS_IPF_NONE && lane == (uint32_t)(__ffs(tpeers) - 1)) atomicAdd(&hits[term], (uint32_t)__popc(tpeers));
  }
}

// K1k ipf_class_kernel — the verdict of every (filter class, node): a thread per node, grid.y over the classes in chunks
// (class0 + blockIdx.y), the class's entries with their keys and slots in shared memory.  Steps 1-4 of bsched.h in
// order, the first failure deciding.  One ballot per warp and plane: bits [3][n_classes][Wg] = pass, failed at step 1
// (E), failed at step 3 (A); a failing node with neither E nor A failed at step 4 (N).  Padding nodes get 0 everywhere.
__global__ void __launch_bounds__(IPF_THREADS) ipf_class_kernel(IpfPods pc, IpfTopo tp, const uint32_t* mbits,
                                                                 const uint32_t* obits, const uint32_t* hits,
                                                                 uint32_t* bits, uint32_t Wg, uint32_t class0) {
  __shared__ uint32_t s_key[BS_IPF_CLASS_MAX], s_off[BS_IPF_CLASS_MAX];
  __shared__ uint8_t s_role[BS_IPF_CLASS_MAX];
  __shared__ uint32_t s_n_aff, s_n_anti, s_hit;
  const uint32_t c = class0 + blockIdx.y;
  if (c >= pc.n_classes) return;   // block-uniform
  const uint32_t o0 = pc.offset[c], n = pc.offset[c + 1] - o0;
  if (threadIdx.x == 0) s_n_aff = s_n_anti = s_hit = 0;
  __syncthreads();
  if (threadIdx.x < n) {
    const uint32_t t = pc.term[o0 + threadIdx.x];
    const uint8_t r = pc.role[o0 + threadIdx.x];
    s_key[threadIdx.x] = tp.term_key[t];
    s_off[threadIdx.x] = tp.term_off[t];
    s_role[threadIdx.x] = r;
    if (r == BS_IPF_AFFINITY) {
      atomicAdd(&s_n_aff, 1u);
      if (hits[t]) atomicOr(&s_hit, 1u);
    } else if (r == BS_IPF_ANTI) {
      atomicAdd(&s_n_anti, 1u);
    }
  }
  __syncthreads();
  const uint32_t i = blockIdx.x * IPF_THREADS + threadIdx.x, lane = threadIdx.x & 31;
  auto present = [&](const uint32_t* plane, uint32_t k, bool& carried) {
    const uint32_t v = tp.topo[(size_t)s_key[k] * tp.n_nodes + i];
    carried = v != BS_TOPO_NONE;
    if (!carried) return false;
    const uint64_t slot = (uint64_t)s_off[k] + v;
    return ((plane[slot >> 5] >> (slot & 31)) & 1u) != 0;
  };
  bool fe = false, fa = false, fn = false;
  if (i < tp.n_nodes) {
    bool carried;
    for (uint32_t k = 0; k < n && !fe; ++k)   // 1. existing pods' anti-affinity
      fe = s_role[k] == BS_IPF_EXISTING && present(obits, k, carried);
    if (!fe && s_n_aff) {                      // 3. every affinity term has a matching pod in n's topology
      bool all = true;
      for (uint32_t k = 0; k < n && all; ++k)
        if (s_role[k] == BS_IPF_AFFINITY) all = present(mbits, k, carried);
      fa = !all && !(s_hit == 0 && pc.self_match[c]);
    }
    if (!fe && !fa && s_n_anti)                // 4. no anti-affinity term has a matching pod in n's topology
      for (uint32_t k = 0; k < n && !fn; ++k) fn = s_role[k] == BS_IPF_ANTI && present(mbits, k, carried);
  }
  const bool pass = i < tp.n_nodes && !(fe || fa || fn);
  const uint32_t wp = __ballot_sync(0xffffffffu, pass), we = __ballot_sync(0xffffffffu, fe),
                 wa = __ballot_sync(0xffffffffu, fa);
  if (lane == 0 && (i >> 5) < Wg) {
    const size_t plane = (size_t)pc.n_classes * Wg, at = (size_t)c * Wg + (i >> 5);
    bits[at] = wp;
    bits[plane + at] = we;
    bits[2 * plane + at] = wa;
  }
}

#endif  // BS_KERNELS_HELPERS_ONLY

}  // namespace bsk
