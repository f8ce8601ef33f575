// Cluster (latency) mode of the beam kernel: depth 1.
#include "uis_launch.cuh"
namespace uis {
bool launch_beam_cluster(int H, int D, const BeamParams& p, int ctas, int cluster, unsigned smem, cudaStream_t st,
                         cudaError_t* err) {
  if (p.depth != 1) return false;
  return with_shape(LatencyShapes{}, H, D, [&](auto s) {
    using S = decltype(s);
    cudaLaunchAttribute attr{};
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = (unsigned)cluster;
    attr.val.clusterDim.y = 1;
    attr.val.clusterDim.z = 1;
    *err = launch_with_attr(uis_beam_kernel<S::H, S::D, false, 1>, p, ctas, Cfg<S::H, S::D, kCPCluster>::BLOCK, smem, st,
                            attr);
  });
}
}  // namespace uis
