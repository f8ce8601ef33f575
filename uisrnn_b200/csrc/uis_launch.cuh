// Kernel launchers, one translation unit per (kernel family, shape group) so that nvcc compiles
// the heavy template instantiations in parallel (`--threads 0`).  uis_api.cu only sees these.
#pragma once
#include <cuda_runtime.h>
#include "uis_beam.cuh"

namespace uis {
// each returns false if (H, D) is not one of its shapes; *err receives the CUDA status otherwise
bool launch_beam_large(int H, int D, const BeamParams& p, int ctas, unsigned smem, cudaStream_t st, cudaError_t* err);
bool launch_beam_small(int H, int D, const BeamParams& p, int ctas, unsigned smem, cudaStream_t st, cudaError_t* err);
// cluster (latency) mode: `ctas` = clusters * cluster; false if the shape has no cluster instantiation
bool launch_beam_cluster(int H, int D, const BeamParams& p, int ctas, int cluster, unsigned smem, cudaStream_t st,
                         cudaError_t* err);
unsigned beam_cluster_smem(int H, int D, int B, int Kcap);
// stationary-weights (latency) mode: `ctas` = groups * kStatGroup, cooperative launch; false if the shape has no instantiation
bool launch_beam_stat(int H, int D, const BeamParams& p, int ctas, unsigned smem, cudaStream_t st, cudaError_t* err);
unsigned beam_stat_smem(int H, int D, int B, int Kcap);
// tensor-core pass (uis_beam_tc.cuh), N = columns per pass (32 or 48)
bool beam_tc_supported(int H, int D, int N);
unsigned beam_tc_smem(int H, int D, int N, int B, int Kcap, int G);
bool launch_beam_tc(int H, int D, int N, const BeamParams& p, int ctas, unsigned smem, cudaStream_t st, cudaError_t* err);
bool launch_tree_large(int H, int D, const BeamParams& p, int ctas, unsigned smem, cudaStream_t st, cudaError_t* err);
bool launch_tree_small(int H, int D, const BeamParams& p, int ctas, unsigned smem, cudaStream_t st, cudaError_t* err);
// the same shapes with the tree-sized arrays in a device-memory arena (p.tree_arena)
bool launch_tree_spill_large(int H, int D, const BeamParams& p, int ctas, unsigned smem, cudaStream_t st, cudaError_t* err);
bool launch_tree_spill_small(int H, int D, const BeamParams& p, int ctas, unsigned smem, cudaStream_t st, cudaError_t* err);

template <class Kern>
inline cudaError_t launch_with_smem(Kern kern, const BeamParams& p, int ctas, int block, unsigned smem, cudaStream_t st) {
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  kern<<<ctas, block, smem, st>>>(p);
  return cudaGetLastError();
}
}  // namespace uis
