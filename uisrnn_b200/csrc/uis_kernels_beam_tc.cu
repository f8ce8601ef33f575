// Tensor-core (wgmma) variant of the beam kernel: look_ahead 1, depth 1, shapes whose weight matrices tile by 128 rows.
#include "uis_launch.cuh"
namespace uis {
namespace {
template <int H, int D, int N>
cudaError_t launch_tc(const BeamParams& p, int ctas, unsigned smem, cudaStream_t st) {
  BeamParams q = p;
  q.tc_layout = make_layout<H, D, kCPBeam, false, N>(p.B, p.Kcap, p.G);
  return launch_with_smem(uis_beam_kernel<H, D, false, false, N>, q, ctas, Cfg<H, D>::BLOCK, smem, st);
}
}  // namespace

bool launch_beam_tc(int H, int D, int N, const BeamParams& p, int ctas, unsigned smem, cudaStream_t st, cudaError_t* err) {
  bool have = false;
  with_shape(TcShapes{}, H, D, [&](auto s) {
    using S = decltype(s);
    have = with_tc_columns(N, [&](auto n) { *err = launch_tc<S::H, S::D, decltype(n)::value>(p, ctas, smem, st); });
  });
  return have;
}
}  // namespace uis
