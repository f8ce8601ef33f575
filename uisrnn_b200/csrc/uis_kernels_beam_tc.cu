// Tensor-core (wgmma) variant of the beam kernel: look_ahead 1, depth 1, shapes whose weight matrices tile by 128 rows.
#include "uis_launch.cuh"
namespace uis {
namespace {
template <int H, int D, int N>
cudaError_t launch_tc(const BeamParams& p, int ctas, unsigned smem, cudaStream_t st) {
  auto kern = uis_beam_kernel<H, D, false, false, N>;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  BeamParams q = p;
  q.tc_layout = make_layout<H, D, kCPBeam, false, N>(p.B, p.Kcap, p.G);
  kern<<<ctas, Cfg<H, D>::BLOCK, smem, st>>>(q);
  return cudaGetLastError();
}
}  // namespace

bool beam_tc_supported(int H, int D, int N) {
  return ((H == 512 && D == 256) || (H == 256 && D == 128)) && (N == 32 || N == 48);
}
unsigned beam_tc_smem(int H, int D, int N, int B, int Kcap, int G) {
  if (H == 512 && D == 256 && N == 48) return make_layout<512, 256, kCPBeam, false, 48>(B, Kcap, G).total;
  if (H == 512 && D == 256 && N == 32) return make_layout<512, 256, kCPBeam, false, 32>(B, Kcap, G).total;
  if (H == 256 && D == 128 && N == 48) return make_layout<256, 128, kCPBeam, false, 48>(B, Kcap, G).total;
  if (H == 256 && D == 128 && N == 32) return make_layout<256, 128, kCPBeam, false, 32>(B, Kcap, G).total;
  return 0xffffffffu;
}
bool launch_beam_tc(int H, int D, int N, const BeamParams& p, int ctas, unsigned smem, cudaStream_t st, cudaError_t* err) {
  if (H == 512 && D == 256 && N == 48) { *err = launch_tc<512, 256, 48>(p, ctas, smem, st); return true; }
  if (H == 512 && D == 256 && N == 32) { *err = launch_tc<512, 256, 32>(p, ctas, smem, st); return true; }
  if (H == 256 && D == 128 && N == 48) { *err = launch_tc<256, 128, 48>(p, ctas, smem, st); return true; }
  if (H == 256 && D == 128 && N == 32) { *err = launch_tc<256, 128, 32>(p, ctas, smem, st); return true; }
  return false;
}
}  // namespace uis
