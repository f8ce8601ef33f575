// Kernel launchers, one translation unit per (kernel family, shape group) so that nvcc compiles the heavy template
// instantiations in parallel (`--threads 0`).  uis_api.cu only sees these.
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <utility>

#include "uis_beam.cuh"

namespace uis {
// The instantiated kernel shapes (hidden H, observation dim D), smallest first.  A model of another size runs
// zero-padded in the smallest listed shape that holds it (uis_model_create).
constexpr int kShapes[][2] = {{128, 64}, {256, 128}, {512, 256}, {1024, 512}};
template <int H_, int D_> struct Shape { static constexpr int H = H_, D = D_; };

// Subsets of kShapes, by index.  The FFMA beam and tree kernels exist at every shape, their launchers split over two
// translation units each (small / large); the tensor-core kernel needs weight matrices that tile by 128 rows; the
// cluster and stationary-weights (latency) modes exist at (512, 256) only.
constexpr size_t kNumShapes = sizeof(kShapes) / sizeof(kShapes[0]);
using AllShapes = std::make_index_sequence<kNumShapes>;
using SmallShapes = std::index_sequence<0, 1>;
using LargeShapes = std::index_sequence<2, 3>;
using TcShapes = std::index_sequence<1, 2>;
using LatencyShapes = std::index_sequence<2>;
static_assert(SmallShapes::size() + LargeShapes::size() == kNumShapes, "every shape has FFMA and tree launchers");

// Calls f(Shape<H, D>{}) if (H, D) is a shape of `subset`; false if it is not.
template <size_t... I, class F>
bool with_shape(std::index_sequence<I...>, int H, int D, F&& f) {
  return ((H == kShapes[I][0] && D == kShapes[I][1] && (f(Shape<kShapes[I][0], kShapes[I][1]>{}), true)) || ...);
}

constexpr unsigned kSmemCap = 227u * 1024u;  // dynamic shared memory per CTA on sm_90a
constexpr unsigned kNoKernel = 0xffffffffu;   // the shared memory of a kernel that does not exist at a shape

// The beam kernels a predict() call can launch (uis_api.cu: kernel_smem, launch_kernel).
enum class Kernel {
  Beam,        // FFMA weight pass, G lanes per CTA (uis_beam.cuh)
  Cluster,     // latency mode: a thread-block cluster of 2/4/8 CTAs per utterance, k-split weight passes
  Stat,        // latency mode: kStatGroup CTAs per utterance keep the weights in shared memory (uis_beam_stat.cuh)
  TensorCore,  // wgmma weight pass over kTcColumns columns (uis_beam_tc.cuh)
  Tree,        // look_ahead >= 2, the candidate tree in shared memory (uis_beam_tree.cuh)
  TreeSpill,   // look_ahead >= 2, the tree-sized arrays in a device-memory arena (p.tree_arena)
};

// The implementations of launch_kernel.  Each returns false if (H, D) is not one of its shapes (or, for the latency
// modes, p.depth is not 1); *err receives the CUDA status of the launch otherwise.
bool launch_beam_small(int H, int D, const BeamParams& p, int ctas, unsigned smem, cudaStream_t st, cudaError_t* err);
bool launch_beam_large(int H, int D, const BeamParams& p, int ctas, unsigned smem, cudaStream_t st, cudaError_t* err);
// `ctas` = clusters * cluster
bool launch_beam_cluster(int H, int D, const BeamParams& p, int ctas, int cluster, unsigned smem, cudaStream_t st,
                         cudaError_t* err);
// `ctas` = groups * kStatGroup, cooperative launch
bool launch_beam_stat(int H, int D, const BeamParams& p, int ctas, unsigned smem, cudaStream_t st, cudaError_t* err);
bool launch_beam_tc(int H, int D, const BeamParams& p, int ctas, unsigned smem, cudaStream_t st, cudaError_t* err);
bool launch_tree_small(int H, int D, bool spill, const BeamParams& p, int ctas, unsigned smem, cudaStream_t st,
                       cudaError_t* err);
bool launch_tree_large(int H, int D, bool spill, const BeamParams& p, int ctas, unsigned smem, cudaStream_t st,
                       cudaError_t* err);

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
  float* scores;                // [configs][score_stride]  neg_likelihood of utterance u at [config][u]
  float* frame_out;             // [configs][frame_stride]  per-frame increments of row r at [config][r] (may be null)
  // Row strides of the two outputs: U and rows for a whole call; a group of a call scored in groups of utterances
  // writes its columns of the call's arrays, whose rows are the whole call's U and rows
  int score_stride;
  long long frame_stride;
  int* blocks;                  // [rows] reduce kernel scratch: block counts of utterance u's clusters at row_off[u]
  // A plan made on the device (score_plan): {chains, queued, max_k} in device memory, written by the plan kernels
  // earlier on the stream.  The kernels read `chains` / `queued` from here; the two fields above then only bound the
  // launch grids (chains <= rows, queued <= rows / 2).  nullptr for a host plan.
  const int* counts;
};
unsigned score_smem(int H, int D);  // kNoKernel if (H, D) is not an instantiated shape
// the three kernels of a score call, in order: chains (Gaussian terms of every visit after the first, C::CP = beam_cp
// columns per pass), first visits (mean0 against every chain's first frame), reduce (per utterance, once per config of a
// sweep: the first two do not depend on the decoding parameters); false if (H, D) is not an instantiated shape
bool launch_score_chains(int H, int D, const ScoreParams& sp, int ctas, cudaStream_t st, cudaError_t* err);
bool launch_score_first(int H, int D, const ScoreParams& sp, cudaStream_t st, cudaError_t* err);
cudaError_t launch_score_reduce(const ScoreParams& sp, int cfg, cudaStream_t st);

// The chain plan of a score call with arbitrary int64 ids per frame (uis_score_device_ids), made on the device: the
// plan plan_chains (uis_api.cu) makes from the canonical labels, with no read-back.  The (id, frame) pairs are sorted
// stably by id, then by utterance, so each run of equal ids is one chain with its frames in order; the first frames of
// the runs, scanned in frame order, give the canonical labels and the chain ids (utterance base + canonical label); the
// chain ids are sorted stably by descending run length.  Outputs: labels [rows] (and labels_out, may be null) the
// canonical labels; chain_off [rows + 1] (entries past the last chain hold rows); chain_rows [rows]; counts [3] =
// {chains, queued (chains of length >= 2), max_k (most clusters in one utterance)}.  row_off: device [U + 1].
// ws: score_plan_bytes(rows, U) bytes of device scratch.  Everything is enqueued on `st`.  rows <= INT_MAX - 1.
size_t score_plan_bytes(long long rows, int U);
constexpr int kScorePlanLaunches = 13;  // score_plan's kernels and CUB calls (uis_stats.kernel_launches counts each once)
cudaError_t score_plan(const long long* ids, const long long* row_off, int U, long long rows, void* ws, size_t ws_bytes,
                       int* labels, int* labels_out, long long* chain_off, long long* chain_rows, int* counts,
                       int num_sms, cudaStream_t st);

template <class Kern, class Params>
inline cudaError_t launch_with_smem(Kern kern, const Params& p, int ctas, int block, unsigned smem, cudaStream_t st) {
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  kern<<<ctas, block, smem, st>>>(p);
  return cudaGetLastError();
}

// The same with one launch attribute (cudaLaunchKernelEx): a thread-block cluster dimension or a cooperative launch.
template <class Kern>
inline cudaError_t launch_with_attr(Kern kern, const BeamParams& p, int ctas, int block, unsigned smem, cudaStream_t st,
                                    const cudaLaunchAttribute& attr) {
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3((unsigned)ctas);
  cfg.blockDim = dim3((unsigned)block);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute a = attr;
  cfg.attrs = &a;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kern, p);
}
}  // namespace uis
