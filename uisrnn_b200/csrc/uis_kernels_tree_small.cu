#include "uis_launch.cuh"
#include "uis_beam_tree.cuh"
namespace uis {
bool launch_tree_small(int H, int D, const BeamParams& p, int ctas, unsigned smem, cudaStream_t st, cudaError_t* err) {
  if (H == 256 && D == 128) {
    using C = Cfg<256, 128, tree_cp<256>()>;
    *err = p.depth > 1 ? launch_with_smem(uis_beam_tree_kernel<256, 128, true>, p, ctas, C::BLOCK, smem, st)
                       : launch_with_smem(uis_beam_tree_kernel<256, 128, false>, p, ctas, C::BLOCK, smem, st);
    return true;
  }
  if (H == 128 && D == 64) {
    using C = Cfg<128, 64, tree_cp<128>()>;
    *err = p.depth > 1 ? launch_with_smem(uis_beam_tree_kernel<128, 64, true>, p, ctas, C::BLOCK, smem, st)
                       : launch_with_smem(uis_beam_tree_kernel<128, 64, false>, p, ctas, C::BLOCK, smem, st);
    return true;
  }
  return false;
}
}  // namespace uis
