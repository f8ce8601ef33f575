#include "uis_launch.cuh"
#include "uis_beam_tree.cuh"
namespace uis {
template <int H, int D, bool SPILL>
static cudaError_t launch_tree(const BeamParams& p, int ctas, unsigned smem, cudaStream_t st) {
  using C = Cfg<H, D, tree_cp<H>()>;
  return p.depth > 1 ? launch_with_smem(uis_beam_tree_kernel<H, D, true, SPILL>, p, ctas, C::BLOCK, smem, st)
                     : launch_with_smem(uis_beam_tree_kernel<H, D, false, SPILL>, p, ctas, C::BLOCK, smem, st);
}

bool launch_tree_small(int H, int D, const BeamParams& p, int ctas, unsigned smem, cudaStream_t st, cudaError_t* err) {
  if (H == 256 && D == 128) { *err = launch_tree<256, 128, false>(p, ctas, smem, st); return true; }
  if (H == 128 && D == 64) { *err = launch_tree<128, 64, false>(p, ctas, smem, st); return true; }
  return false;
}

bool launch_tree_spill_small(int H, int D, const BeamParams& p, int ctas, unsigned smem, cudaStream_t st, cudaError_t* err) {
  if (H == 256 && D == 128) { *err = launch_tree<256, 128, true>(p, ctas, smem, st); return true; }
  if (H == 128 && D == 64) { *err = launch_tree<128, 64, true>(p, ctas, smem, st); return true; }
  return false;
}
}  // namespace uis
