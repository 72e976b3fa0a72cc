// replay_ipf_inst.cu — the IPF builds of replay_kernel (replay.cuh): every node choice with and without HP for one MAXL,
// chosen with -DBS_REPLAY_IPF_MAXL=5, 9 or 16 (build.py compiles the file once per value), so that the 30 builds compile
// in three units in parallel with engine.cu, which keeps the 30 without the filter.
#define BS_KERNELS_HELPERS_ONLY   // kernels.cuh's round kernels live in engine.cu
#include "replay.cuh"

#ifndef BS_REPLAY_IPF_MAXL
#error "compile with -DBS_REPLAY_IPF_MAXL=5, 9 or 16"
#endif

namespace bsk {

template <int MAXL, bool HP>
void launch_replay_ipf(const ReplayArgs& a, bool scored, bool loc, cudaStream_t s) {
  launch_replay_t<MAXL, HP, true>(a, scored, loc, s);
}

template void launch_replay_ipf<BS_REPLAY_IPF_MAXL, false>(const ReplayArgs&, bool, bool, cudaStream_t);
template void launch_replay_ipf<BS_REPLAY_IPF_MAXL, true>(const ReplayArgs&, bool, bool, cudaStream_t);

}  // namespace bsk
