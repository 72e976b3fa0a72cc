// replay_inst.cu — the builds of replay_kernel (replay.cuh), compiled once per slice (build.py, -DBS_REPLAY_SLICE=k for
// k = 0..5) so that the 60 builds compile in parallel with the other units: slice k holds the 10 builds of lane bound 5,
// 9 or 16 (k / 2 = 0, 1, 2) with IPF off (even k) or on (odd k).  engine.cu reaches them through launch_replay_slice.
#define BS_KERNELS_HELPERS_ONLY   // kernels.cuh's round kernels live in engine.cu
#include "replay.cuh"

#ifndef BS_REPLAY_SLICE
#error "compile with -DBS_REPLAY_SLICE=0..5"
#endif

namespace bsk {

template <int MAXL, uint32_t IPF>
void launch_replay_slice(uint32_t build, const ReplayIpfArgs& a, cudaStream_t s) {
  with_flags<REPLAY_IPF>(build % REPLAY_IPF, [&](auto low) {
    constexpr uint32_t B = IPF | decltype(low)::value;
    if constexpr (replay_build_exists(B))
      replay_kernel<MAXL, (B & REPLAY_SCORED) != 0, (B & REPLAY_RATIO) != 0, (B & REPLAY_LOC) != 0,
                    (B & REPLAY_HP) != 0, (B & REPLAY_IPF) != 0><<<1, REPLAY_THREADS, 0, s>>>(a);
  });
}
constexpr int SLICE_MAXL[] = {5, 9, 16};
template void launch_replay_slice<SLICE_MAXL[BS_REPLAY_SLICE / 2], BS_REPLAY_SLICE % 2 * REPLAY_IPF>(
    uint32_t, const ReplayIpfArgs&, cudaStream_t);

}  // namespace bsk
