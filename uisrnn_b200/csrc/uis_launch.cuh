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

// score(): the neg_likelihood of given labellings (uis_kernels_score.cu).  With the labels fixed, every (utterance,
// cluster) pair is an independent chain of GRU steps over that cluster's frames; the chain kernel packs the chains'
// steps into the columns of the FFMA weight pass (run_pass), the reduce kernel adds the per-frame terms.
struct ScoreParams {
  BeamParams b;                 // model, x, gi, log tables, slot pools (P = 2: two slots per column), queue, stats
  const long long* chain_off;   // [chains + 1] offsets into chain_rows; chains longest first
  const long long* chain_rows;  // [rows] every chain's frame rows in frame order
  int chains;                   // chains of the call (one per utterance and cluster)
  int queued;                   // the first `queued` chains (length >= 2) run through the chain kernel
  float* mse;                   // [rows] Gaussian term of a frame against its cluster's mean before that frame
  const int* labels;            // [rows] canonical labels
  float* scores;                // [configs][U]    neg_likelihood
  float* frame_out;             // [configs][rows] per-frame increments (may be null)
  int* blocks;                  // [rows] reduce kernel scratch: block counts of utterance u's clusters at row_off[u]
};
constexpr int score_cp(int H) { return H > 512 ? 8 : kCPBeam; }  // columns per pass (= the FFMA beam kernel's)
unsigned score_smem(int H, int D);
// the three kernels of a score call, in order: chains (Gaussian terms of every visit after the first), first visits
// (mean0 against every chain's first frame), reduce (per utterance, once per config of a sweep: the first two do not
// depend on the decoding parameters); false if (H, D) is not an instantiated shape
bool launch_score_chains(int H, int D, const ScoreParams& sp, int ctas, cudaStream_t st, cudaError_t* err);
bool launch_score_first(int D, const ScoreParams& sp, cudaStream_t st, cudaError_t* err);
cudaError_t launch_score_reduce(const ScoreParams& sp, int cfg, cudaStream_t st);

template <class Kern>
inline cudaError_t launch_with_smem(Kern kern, const BeamParams& p, int ctas, int block, unsigned smem, cudaStream_t st) {
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  kern<<<ctas, block, smem, st>>>(p);
  return cudaGetLastError();
}
}  // namespace uis
