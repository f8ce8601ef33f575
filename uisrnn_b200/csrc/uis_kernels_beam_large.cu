#include "uis_launch.cuh"
namespace uis {
bool launch_beam_large(int H, int D, const BeamParams& p, int ctas, unsigned smem, cudaStream_t st, cudaError_t* err) {
  if (H == 512 && D == 256) {
    *err = p.depth > 1 ? launch_with_smem(uis_beam_kernel<512, 256, true>, p, ctas, Cfg<512, 256>::BLOCK, smem, st)
                       : launch_with_smem(uis_beam_kernel<512, 256, false>, p, ctas, Cfg<512, 256>::BLOCK, smem, st);
    return true;
  }
  if (H == 1024 && D == 512) {  // FFMA engine only (8 columns per pass, beam_cp)
    *err = p.depth > 1 ? launch_with_smem(uis_beam_kernel<1024, 512, true>, p, ctas, Cfg<1024, 512>::BLOCK, smem, st)
                       : launch_with_smem(uis_beam_kernel<1024, 512, false>, p, ctas, Cfg<1024, 512>::BLOCK, smem, st);
    return true;
  }
  return false;
}
}  // namespace uis
