// Stationary-weights (latency) mode of the beam kernel (uis_beam_stat.cuh): depth 1.
#include "uis_launch.cuh"
namespace uis {
bool launch_beam_stat(int H, int D, const BeamParams& p, int ctas, unsigned smem, cudaStream_t st, cudaError_t* err) {
  if (p.depth != 1) return false;
  return with_shape(LatencyShapes{}, H, D, [&](auto s) {
    using S = decltype(s);
    cudaLaunchAttribute attr{};
    attr.id = cudaLaunchAttributeCooperative;  // the groups synchronise through global memory: all CTAs must be co-resident
    attr.val.cooperative = 1;
    *err = launch_with_attr(uis_beam_kernel<S::H, S::D, false, 2>, p, ctas, Cfg<S::H, S::D, kCPCluster>::BLOCK, smem, st,
                            attr);
  });
}
}  // namespace uis
