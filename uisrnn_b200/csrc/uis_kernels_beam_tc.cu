// Tensor-core (wgmma) variant of the beam kernel: look_ahead 1, depth 1, shapes whose weight matrices tile by 128 rows.
#include "uis_launch.cuh"
namespace uis {
bool launch_beam_tc(int H, int D, const BeamParams& p, int ctas, unsigned smem, cudaStream_t st, cudaError_t* err) {
  return with_shape(TcShapes{}, H, D, [&](auto s) {
    using S = decltype(s);
    BeamParams q = p;
    q.tc_layout = make_layout<S::H, S::D, kCPBeam, false, kTcColumns>(p.B, p.Kcap, p.G);
    *err = launch_with_smem(uis_beam_kernel<S::H, S::D, false, false, kTcColumns>, q, ctas, Cfg<S::H, S::D>::BLOCK, smem, st);
  });
}
}  // namespace uis
