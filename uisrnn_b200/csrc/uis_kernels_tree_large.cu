#include "uis_launch.cuh"
#include "uis_beam_tree.cuh"
namespace uis {
template <int H, int D, bool SPILL>
static cudaError_t launch_tree(const BeamParams& p, int ctas, unsigned smem, cudaStream_t st) {
  using C = Cfg<H, D, tree_cp<H>()>;  // 8 columns per pass at (1024, 512) (tree_cp)
  return p.depth > 1 ? launch_with_smem(uis_beam_tree_kernel<H, D, true, SPILL>, p, ctas, C::BLOCK, smem, st)
                     : launch_with_smem(uis_beam_tree_kernel<H, D, false, SPILL>, p, ctas, C::BLOCK, smem, st);
}

bool launch_tree_large(int H, int D, const BeamParams& p, int ctas, unsigned smem, cudaStream_t st, cudaError_t* err) {
  if (H == 512 && D == 256) { *err = launch_tree<512, 256, false>(p, ctas, smem, st); return true; }
  if (H == 1024 && D == 512) { *err = launch_tree<1024, 512, false>(p, ctas, smem, st); return true; }
  return false;
}

bool launch_tree_spill_large(int H, int D, const BeamParams& p, int ctas, unsigned smem, cudaStream_t st, cudaError_t* err) {
  if (H == 512 && D == 256) { *err = launch_tree<512, 256, true>(p, ctas, smem, st); return true; }
  if (H == 1024 && D == 512) { *err = launch_tree<1024, 512, true>(p, ctas, smem, st); return true; }
  return false;
}
}  // namespace uis
