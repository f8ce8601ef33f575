#include "uis_launch.cuh"
namespace uis {
bool launch_beam_small(int H, int D, const BeamParams& p, int ctas, unsigned smem, cudaStream_t st, cudaError_t* err) {
  return with_shape(SmallShapes{}, H, D, [&](auto s) {
    using S = decltype(s);
    *err = p.depth > 1 ? launch_with_smem(uis_beam_kernel<S::H, S::D, true>, p, ctas, Cfg<S::H, S::D>::BLOCK, smem, st)
                       : launch_with_smem(uis_beam_kernel<S::H, S::D, false>, p, ctas, Cfg<S::H, S::D>::BLOCK, smem, st);
  });
}
}  // namespace uis
