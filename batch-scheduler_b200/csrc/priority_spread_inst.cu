// priority_spread_inst.cu — the SPREAD variants of priority_pod_kernel (priority.cuh): every combination of RATIO, PREF
// and LOC for one MAXL, chosen with -DBS_PRIO_SPREAD_MAXL=5, 9 or 16 (build.py compiles the file once per value), so
// that the 24 variants compile in three units in parallel with engine.cu and priority_inst.cu.
#define BS_KERNELS_HELPERS_ONLY   // kernels.cuh's round kernels live in engine.cu
#include "priority.cuh"

#ifndef BS_PRIO_SPREAD_MAXL
#error "compile with -DBS_PRIO_SPREAD_MAXL=5, 9 or 16"
#endif

namespace bsk {

template <int M>
void launch_priority_spread(uint32_t grid, bool ratio, bool pref, bool loc, const PrioritySpreadArgs& a, cudaStream_t s) {
  if (loc) {
    if (pref && ratio) priority_pod_kernel<M, true, true, true, true><<<grid, PRIO_THREADS, 0, s>>>(a);
    else if (pref) priority_pod_kernel<M, false, true, true, true><<<grid, PRIO_THREADS, 0, s>>>(a);
    else if (ratio) priority_pod_kernel<M, true, false, true, true><<<grid, PRIO_THREADS, 0, s>>>(a);
    else priority_pod_kernel<M, false, false, true, true><<<grid, PRIO_THREADS, 0, s>>>(a);
  } else {
    if (pref && ratio) priority_pod_kernel<M, true, true, false, true><<<grid, PRIO_THREADS, 0, s>>>(a);
    else if (pref) priority_pod_kernel<M, false, true, false, true><<<grid, PRIO_THREADS, 0, s>>>(a);
    else if (ratio) priority_pod_kernel<M, true, false, false, true><<<grid, PRIO_THREADS, 0, s>>>(a);
    else priority_pod_kernel<M, false, false, false, true><<<grid, PRIO_THREADS, 0, s>>>(a);
  }
}

template void launch_priority_spread<BS_PRIO_SPREAD_MAXL>(uint32_t, bool, bool, bool, const PrioritySpreadArgs&,
                                                          cudaStream_t);

}  // namespace bsk
