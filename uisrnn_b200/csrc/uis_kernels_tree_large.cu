#include "uis_launch.cuh"
#include "uis_beam_tree.cuh"
namespace uis {
bool launch_tree_large(int H, int D, const BeamParams& p, int ctas, unsigned smem, cudaStream_t st, cudaError_t* err) {
  if (H == 512 && D == 256) {
    using C = Cfg<512, 256, tree_cp<512>()>;
    *err = p.depth > 1 ? launch_with_smem(uis_beam_tree_kernel<512, 256, true>, p, ctas, C::BLOCK, smem, st)
                       : launch_with_smem(uis_beam_tree_kernel<512, 256, false>, p, ctas, C::BLOCK, smem, st);
    return true;
  }
  if (H == 1024 && D == 512) {  // 8 columns per pass (tree_cp)
    using C = Cfg<1024, 512, tree_cp<1024>()>;
    *err = p.depth > 1 ? launch_with_smem(uis_beam_tree_kernel<1024, 512, true>, p, ctas, C::BLOCK, smem, st)
                       : launch_with_smem(uis_beam_tree_kernel<1024, 512, false>, p, ctas, C::BLOCK, smem, st);
    return true;
  }
  return false;
}
}  // namespace uis
