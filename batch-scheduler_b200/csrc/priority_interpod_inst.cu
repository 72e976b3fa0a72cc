// priority_interpod_inst.cu — the IPA variants of priority_pod_kernel (priority.cuh): every combination of RATIO, PREF,
// LOC and SPREAD for one MAXL, chosen with -DBS_PRIO_IPA_MAXL=5, 9 or 16 (build.py compiles the file once per value),
// so that the 48 variants compile in three units in parallel with the other units.
#define BS_KERNELS_HELPERS_ONLY   // kernels.cuh's round kernels live in engine.cu
#include "priority.cuh"

#ifndef BS_PRIO_IPA_MAXL
#error "compile with -DBS_PRIO_IPA_MAXL=5, 9 or 16"
#endif

namespace bsk {
namespace {

template <int M, bool LOC, bool SPREAD>
void launch_ipa(uint32_t grid, bool ratio, bool pref, const PriorityIpaArgs& a, cudaStream_t s) {
  if (pref && ratio) priority_pod_kernel<M, true, true, LOC, SPREAD, true><<<grid, PRIO_THREADS, 0, s>>>(a);
  else if (pref) priority_pod_kernel<M, false, true, LOC, SPREAD, true><<<grid, PRIO_THREADS, 0, s>>>(a);
  else if (ratio) priority_pod_kernel<M, true, false, LOC, SPREAD, true><<<grid, PRIO_THREADS, 0, s>>>(a);
  else priority_pod_kernel<M, false, false, LOC, SPREAD, true><<<grid, PRIO_THREADS, 0, s>>>(a);
}

}  // namespace

template <int M>
void launch_priority_interpod(uint32_t grid, bool ratio, bool pref, bool loc, bool spread, const PriorityIpaArgs& a,
                              cudaStream_t s) {
  if (loc && spread) launch_ipa<M, true, true>(grid, ratio, pref, a, s);
  else if (loc) launch_ipa<M, true, false>(grid, ratio, pref, a, s);
  else if (spread) launch_ipa<M, false, true>(grid, ratio, pref, a, s);
  else launch_ipa<M, false, false>(grid, ratio, pref, a, s);
}

template void launch_priority_interpod<BS_PRIO_IPA_MAXL>(uint32_t, bool, bool, bool, bool, const PriorityIpaArgs&,
                                                         cudaStream_t);

}  // namespace bsk
