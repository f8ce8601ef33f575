// C ABI of libuisrnn_b200.so (see include/uisrnn_b200.h).  Host-side orchestration only:
// weight re-layout at model creation, workspace management, utterance scheduling (longest
// first), kernel launches.  No PyTorch types, no CPU compute fallback: if the kernels are not
// instantiated for a shape the call fails with UIS_ERR_UNSUPPORTED.
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <condition_variable>
#include <mutex>
#include <thread>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <numeric>
#include <string>
#include <vector>

#include "../../include/uisrnn_b200.h"
#include "uis_beam.cuh"
#include "uis_beam_tree.cuh"
#include "uis_launch.cuh"
#include "uis_prepass.cuh"

namespace {
thread_local std::string g_err;
}

namespace uis {
// shared with uis_train.cu
int api_fail(int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  g_err = buf;
  return code;
}
}  // namespace uis

namespace {

template <class... Args>
int fail(int code, const char* fmt, Args... args) {
  return uis::api_fail(code, fmt, args...);
}

#define CU(call)                                                                              \
  do {                                                                                        \
    cudaError_t e_ = (call);                                                                  \
    if (e_ != cudaSuccess)                                                                    \
      return fail(UIS_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, \
                  __LINE__);                                                                  \
  } while (0)

struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  int ensure(size_t bytes) {
    if (bytes <= cap) return 0;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    size_t want = bytes + bytes / 8 + 256;
    cudaError_t e = cudaMalloc(&p, want);
    if (e != cudaSuccess) {
      want = bytes;
      e = cudaMalloc(&p, want);
    }
    if (e != cudaSuccess) return fail(UIS_ERR_NOMEM, "cudaMalloc(%zu) failed: %s", want, cudaGetErrorString(e));
    cap = want;
    return 0;
  }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
  }
  template <class T> T* as() const { return static_cast<T*>(p); }
};

int fetch(std::vector<float>& dst, const float* src, size_t n) {
  dst.resize(n);
  CU(cudaMemcpy(dst.data(), src, n * sizeof(float), cudaMemcpyDefault));
  return 0;
}

int upload(DevBuf& b, const void* src, size_t bytes) {
  if (int rc = b.ensure(bytes)) return rc;
  CU(cudaMemcpy(b.p, src, bytes, cudaMemcpyHostToDevice));
  return 0;
}

std::vector<float> transpose(const std::vector<float>& w, int rows, int cols) {
  std::vector<float> t((size_t)rows * cols);
  for (int r = 0; r < rows; ++r)
    for (int c = 0; c < cols; ++c) t[(size_t)c * rows + r] = w[(size_t)r * cols + c];
  return t;
}

// Host threads that copy the pieces of one staging chunk from the caller's PAGEABLE arrays into pinned memory, side by
// side (a cudaMemcpy from pageable memory is staged by the driver in one thread at ~11 GB/s; several threads reach
// the PCIe rate).  run() hands the same piece list to every worker; worker i copies bytes [total * i / n, total * (i + 1) / n).
struct CopyPiece { const char* src; size_t dst_off, bytes; };
class CopyPool {
 public:
  explicit CopyPool(int n) : n_(n) {
    for (int i = 0; i < n; ++i) th_.emplace_back([this, i] { loop(i); });
  }
  ~CopyPool() {
    { std::lock_guard<std::mutex> lk(mu_); stop_ = true; ++gen_; }
    cv_.notify_all();
    for (auto& t : th_) t.join();
  }
  void run(const std::vector<CopyPiece>* pieces, char* dst, size_t total) {
    { std::lock_guard<std::mutex> lk(mu_); pieces_ = pieces; dst_ = dst; total_ = total; pending_ = n_; ++gen_; }
    cv_.notify_all();
    std::unique_lock<std::mutex> lk(mu_);
    done_.wait(lk, [&] { return pending_ == 0; });
  }
 private:
  void loop(int i) {
    unsigned long long seen = 0;
    for (;;) {
      const std::vector<CopyPiece>* pieces; char* dst; size_t total;
      {
        std::unique_lock<std::mutex> lk(mu_);
        cv_.wait(lk, [&] { return gen_ != seen; });
        seen = gen_;
        if (stop_) return;
        pieces = pieces_; dst = dst_; total = total_;
      }
      const size_t b0 = total * (size_t)i / (size_t)n_, b1 = total * (size_t)(i + 1) / (size_t)n_;
      for (const CopyPiece& p : *pieces) {
        const size_t lo = std::max(b0, p.dst_off), hi = std::min(b1, p.dst_off + p.bytes);
        if (lo < hi) std::memcpy(dst + lo, p.src + (lo - p.dst_off), hi - lo);
      }
      std::lock_guard<std::mutex> lk(mu_);
      if (--pending_ == 0) done_.notify_one();
    }
  }
  int n_;
  std::vector<std::thread> th_;
  std::mutex mu_;
  std::condition_variable cv_, done_;
  const std::vector<CopyPiece>* pieces_ = nullptr;
  char* dst_ = nullptr;
  size_t total_ = 0;
  int pending_ = 0;
  unsigned long long gen_ = 0;
  bool stop_ = false;
};
}  // namespace

struct uis_model {
  int device = 0, D = 0, H = 0, depth = 1, num_sms = 0;  // D, H: the kernel shape the model runs in
  int D_user = 0, H_user = 0;  // the caller's shape (<= D, H): smaller models are zero-padded into the next kernel shape
  double p0 = 0, alpha = 0;
  // weights, k-major
  DevBuf wih_t, whh_t, w1_t, w2_t, bih, bhh, b1, b2, wvec, mean0, hidden0;
  DevBuf wih_up_t;  // [depth-1][H][3H]; whh_t is [depth][H][3H]; bih / bhh are [depth][3H]
  // tensor-core pass (uis_beam_tc.cuh): fp16 hi/lo planes of [W_hh; W1; W2] behind a tensor map, scales
  DevBuf tc_planes, tc_scratch, stat_bar, stat_scratch;
  alignas(64) CUtensorMap tc_map;
  bool tc_ready = false;
  float tc_sh = 0, tc_sa = 0, tc_inv_hh = 0, tc_inv_1 = 0, tc_inv_2 = 0;
  // log tables: logn [log_cap] is shared; the decoding-parameter tables (LogTables) of the model's own values and of
  // the last sweep are kept apart, so that a sweep never rebuilds the tables of a plain call
  DevBuf logn;
  int log_cap = 0;
  struct LogTables {
    DevBuf tot, cfg;          // [configs][cap] log(i + crp_alpha); [configs][3] log(p0), log(1 - p0), log(crp_alpha)
    std::vector<double> key;  // (crp_alpha, transition_bias) of every config the tables hold
    int cap = 0;
  } own_logs, sweep_logs;
  // workspace
  DevBuf x64, x32, gi, row_off, order, pool_mean, pool_hidden, pool_mse, bp, queue_stats, labels, status;
  DevBuf spk_bound, spk_out;  // bounded calls only: [U][2] speaker bounds; [U] speaker counts (host-buffer entry point)
  DevBuf nb_scores, nb_speakers, nb_count;  // N-best calls, host-buffer entry point: [U][n_best], [U][n_best], [U]
  DevBuf tree_arena;  // look-ahead spill kernel: [spill CTAs][make_tree_arena(..).total]
  // score calls (uis_kernels_score.cu): chain plan, per-frame Gaussian terms, reduce scratch, host entry's outputs
  DevBuf sc_chain_off, sc_chain_rows, sc_mse, sc_blocks, sc_out;
  DevBuf sc_counts, sc_plan;  // device-planned score calls: {chains, queued, max_k, -} per group; the plan kernels' scratch
  DevBuf dbg_win, dbg_score, dbg_off, dbg_final_scores, dbg_final_k, dbg_best_mean, dbg_best_hidden,
      dbg_best_blocks;
  // last call
  uis_stats stats{};
  int last_U = 0;
  bool last_tree_spill = false;  // the last call ran the look-ahead spill kernel (its caps name the arena in errors)
  bool last_score = false;       // the last call was a score call (two counters, no per-utterance status)
  bool last_score_counts = false;  // ... whose chains were planned on the device: max_k is in sc_counts
  // every call records ev_done on its stream after its last work, and the next call's stream waits for it: a call on
  // another stream must not overwrite the workspace while the previous call's kernels still read it
  cudaEvent_t ev_done = nullptr;
  bool done_recorded = false;
  int last_spill_ni = 0, last_spill_nlf = 0;
  size_t last_spill_budget = 0;
  cudaStream_t last_stream = nullptr;
  bool stats_pending = false;
  // before prepass, after prepass, after beam kernel: three per group of the last call that launched kernels
  // (last_groups of them; a call decoded or scored in groups adds up their times)
  std::vector<cudaEvent_t> ev = std::vector<cudaEvent_t>(3, nullptr);
  int last_groups = 1;
  // host-buffer path (uis_predict): the float64 rows travel in chunks through a small ring of staging slots on a
  // copy stream of their own, so the H2D copy of chunk c + 1 runs under the cast + input projection of chunk c and
  // the fp64 staging is O(chunk), not O(input); labels come back in ONE copy into pinned memory
  cudaStream_t copy_stream = nullptr;
  static constexpr int kSlots = 3;
  cudaEvent_t ev_copied[kSlots] = {nullptr, nullptr, nullptr}, ev_free[kSlots] = {nullptr, nullptr, nullptr};
  cudaEvent_t ev_h2d[2] = {nullptr, nullptr};
  cudaEvent_t ev_pipe = nullptr;  // compute stream, before the first cast
  int32_t* labels_pin = nullptr;
  size_t labels_pin_cap = 0;
  // pageable inputs: pinned staging ring (kSlots chunks) filled by host threads, one DMA per chunk
  char* pin_stage = nullptr;
  size_t pin_stage_cap = 0;
  cudaEvent_t ev_dma[kSlots] = {nullptr, nullptr, nullptr};
  CopyPool* copy_pool = nullptr;
};

namespace {

// ---- the kernel variants (uis::Kernel, uis_launch.cuh): shared memory and launch ----------------------------------

// Shared memory of kernel k at the model's shape for the sizes in p (B, Kcap, G; the tree kernels: L, node_cap,
// leaf_cap, P).  uis::kNoKernel if the shape has no such kernel.
unsigned kernel_smem(const uis_model* m, uis::Kernel k, const uis::BeamParams& p) {
  using namespace uis;
  unsigned smem = kNoKernel;
  switch (k) {
    case Kernel::Beam:
      with_shape(AllShapes{}, m->H, m->D, [&](auto s) {
        using S = decltype(s);
        smem = make_layout<S::H, S::D, beam_cp<S::H>()>(p.B, p.Kcap, p.G).total;
      });
      break;
    case Kernel::Cluster:
      with_shape(LatencyShapes{}, m->H, m->D, [&](auto s) {
        using S = decltype(s);
        smem = make_layout<S::H, S::D, kCPCluster, true>(p.B, p.Kcap, p.G).total;
      });
      break;
    case Kernel::Stat:
      with_shape(LatencyShapes{}, m->H, m->D, [&](auto s) {
        using S = decltype(s);
        smem = make_layout<S::H, S::D, kCPCluster, false, 0, true>(p.B, p.Kcap, p.G).total;
      });
      break;
    case Kernel::TensorCore:
      with_shape(TcShapes{}, m->H, m->D, [&](auto s) {
        using S = decltype(s);
        smem = make_layout<S::H, S::D, kCPBeam, false, kTcColumns>(p.B, p.Kcap, p.G).total;
      });
      break;
    case Kernel::Tree:
      with_shape(AllShapes{}, m->H, m->D, [&](auto s) {
        using S = decltype(s);
        smem = make_tree_layout<S::H, S::D>(p.B, p.Kcap, p.L, p.node_cap, p.leaf_cap, p.P).total;
      });
      break;
    case Kernel::TreeSpill:  // the tree-sized arrays live in p.tree_arena: shared memory holds the rest and a scratch
      with_shape(AllShapes{}, m->H, m->D, [&](auto s) {
        smem = make_tree_layout<decltype(s)::H, decltype(s)::D>(p.B, p.Kcap, p.L, 0, 0, 0).total + kTreeSpillScratch;
      });
      break;
  }
  return smem;
}

// The sizes the shared memory of a look_ahead-1 kernel depends on.
uis::BeamParams beam_sizes(int B, int Kcap, int G) {
  uis::BeamParams p{};
  p.B = B; p.Kcap = Kcap; p.G = G;
  return p;
}

// Launches kernel k at the model's shape on `ctas` CTAs (Kernel::Cluster: `cluster` CTAs per cluster).  false if the
// shape has no such kernel; *err = the launch status otherwise.
bool launch_kernel(const uis_model* m, uis::Kernel k, const uis::BeamParams& p, int ctas, int cluster, unsigned smem,
                   cudaStream_t st, cudaError_t* err) {
  const int H = m->H, D = m->D;
  switch (k) {
    case uis::Kernel::Beam:
      return uis::launch_beam_large(H, D, p, ctas, smem, st, err) || uis::launch_beam_small(H, D, p, ctas, smem, st, err);
    case uis::Kernel::Cluster: return uis::launch_beam_cluster(H, D, p, ctas, cluster, smem, st, err);
    case uis::Kernel::Stat: return uis::launch_beam_stat(H, D, p, ctas, smem, st, err);
    case uis::Kernel::TensorCore: return uis::launch_beam_tc(H, D, p, ctas, smem, st, err);
    case uis::Kernel::Tree:
    case uis::Kernel::TreeSpill: {
      const bool spill = k == uis::Kernel::TreeSpill;
      return uis::launch_tree_large(H, D, spill, p, ctas, smem, st, err) ||
             uis::launch_tree_small(H, D, spill, p, ctas, smem, st, err);
    }
  }
  return false;
}

// ---- model creation ----------------------------------------------------------------------------------------------

typedef CUresult (*TensorMapEncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                      const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                      CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// largest power of two s with bound * s <= 2^14 (fp16 keeps 11 significant bits down to 2^-14; |hi| stays < 65504)
float tc_pow2_scale(double bound) {
  if (!(bound > 0.0) || !std::isfinite(bound)) return 0.f;
  int e = 0;
  std::frexp(16384.0 / bound, &e);   // 16384 / bound = f * 2^e, f in [0.5, 1)
  e -= 1;                            // 2^e <= 16384 / bound
  if (e > 40) e = 40;
  if (e < -40) return 0.f;
  return std::ldexp(1.0f, e);
}

// Splits w * scale into fp16 hi + lo (22 significant bits) -- the A operand planes of the wgmma pass.  Returns the
// largest share of a row's sum |w * scale| that the split loses, sum_j |hi + lo - w * scale| over sum_j |w * scale|: the
// relative error the planes add to that row's dot product with a uniformly bounded operand.
double tc_split(const std::vector<float>& w, int cols, float scale, __half* hi, __half* lo) {
  double worst = 0;
  for (size_t r0 = 0; r0 < w.size(); r0 += cols) {
    double lost = 0, mass = 0;
    for (size_t i = r0; i < r0 + cols; ++i) {
      const float v = w[i] * scale;
      const __half h = __float2half_rn(v);
      hi[i] = h;
      lo[i] = __float2half_rn(v - __half2float(h));
      lost += std::fabs((double)__half2float(h) + (double)__half2float(lo[i]) - (double)v);
      mass += std::fabs((double)v);
    }
    if (mass > 0) worst = std::max(worst, lost / mass);
  }
  return worst;
}

// w_hh [3H,H], w1 [H,H], w2 [D,H] are the row-major (= K-major) PyTorch tensors; hidden0 [H] = CoreRNN(0, h0).
// Leaves tc_ready false (the FFMA kernels serve the model) when the shape does not tile, a bound is not finite or
// clamps, or a weight matrix's split loses more than kTcSplitLoss of some row's sum |w * scale| (tc_split): that
// happens when a few weights far above the rest set the matrix's scale and leave the others' lo halves subnormal.
// 2^-20 is below the ~2^-19.5 that a 512-term fp32 FMA chain typically loses relative to its sum of |terms|.  Uniform
// (512, 512) weights lose 2^-25.0; with one entry 2^17 times their largest 2^-21.3 (tensor cores), 2^24 times 2^-14.3
// (FFMA).
constexpr double kTcSplitLoss = 0x1p-20;
int tc_prepare(uis_model* m, const std::vector<float>& w_hh, const std::vector<float>& w1, const std::vector<float>& b1,
               const std::vector<float>& w2, const std::vector<float>& hidden0) {
  const int H = m->H, D = m->D;
  m->tc_ready = false;
  if (m->depth != 1 || kernel_smem(m, uis::Kernel::TensorCore, uis::BeamParams{}) == uis::kNoKernel) return 0;
  auto maxabs = [](const std::vector<float>& v) { double a = 0; for (float x : v) a = std::max(a, (double)std::fabs(x)); return a; };
  // |h'| <= max(1, |h|) by induction (h' is a convex combination of h and tanh(.)), starting from hidden0
  const double hmax = std::max(1.0, maxabs(hidden0));
  double amax = 0;  // a = relu(W1 h' + b1):  |a_i| <= |b1_i| + hmax * sum_j |W1_ij|
  for (int i = 0; i < H; ++i) {
    double srow = 0;
    for (int j = 0; j < H; ++j) srow += std::fabs(w1[(size_t)i * H + j]);
    amax = std::max(amax, std::fabs((double)b1[i]) + hmax * srow);
  }
  const float s_hh = tc_pow2_scale(maxabs(w_hh)), s_1 = tc_pow2_scale(maxabs(w1)), s_2 = tc_pow2_scale(maxabs(w2));
  const float s_h = tc_pow2_scale(hmax), s_a = tc_pow2_scale(std::max(amax, 1e-30));
  if (s_hh == 0.f || s_1 == 0.f || s_2 == 0.f || s_h == 0.f || s_a == 0.f) return 0;
  const size_t rows = (size_t)3 * H + H + D, n = rows * H;
  std::vector<__half> planes(2 * n);  // [plane 0 = lo | plane 1 = hi][rows][H]
  double lost = tc_split(w_hh, H, s_hh, planes.data() + n, planes.data());
  {
    std::vector<__half> hi((size_t)H * H), lo((size_t)H * H);
    lost = std::max(lost, tc_split(w1, H, s_1, hi.data(), lo.data()));
    std::copy(lo.begin(), lo.end(), planes.begin() + (size_t)3 * H * H);
    std::copy(hi.begin(), hi.end(), planes.begin() + n + (size_t)3 * H * H);
  }
  {
    std::vector<__half> hi((size_t)D * H), lo((size_t)D * H);
    lost = std::max(lost, tc_split(w2, H, s_2, hi.data(), lo.data()));
    std::copy(lo.begin(), lo.end(), planes.begin() + (size_t)4 * H * H);
    std::copy(hi.begin(), hi.end(), planes.begin() + n + (size_t)4 * H * H);
  }
  if (!(lost <= kTcSplitLoss)) return 0;
  if (int r = upload(m->tc_planes, planes.data(), planes.size() * sizeof(__half))) return r;
  TensorMapEncodeFn encode = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", reinterpret_cast<void**>(&encode), cudaEnableDefault, &qres) !=
          cudaSuccess || !encode || qres != cudaDriverEntryPointSuccess) {
    (void)cudaGetLastError();
    return 0;  // driver without tensor maps: the FFMA kernels serve the model
  }
  const cuuint64_t gdim[2] = {(cuuint64_t)H, (cuuint64_t)(2 * rows)};
  const cuuint64_t gstr[1] = {(cuuint64_t)H * 2};
  const cuuint32_t box[2] = {64, 128};
  const cuuint32_t estr[2] = {1, 1};
  if (encode(&m->tc_map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, m->tc_planes.p, gdim, gstr, box, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
    return 0;
  m->tc_sh = s_h; m->tc_sa = s_a;
  m->tc_inv_hh = 1.0f / (s_hh * s_h); m->tc_inv_1 = 1.0f / (s_1 * s_h); m->tc_inv_2 = 1.0f / (s_2 * s_a);
  m->tc_ready = true;
  return 0;
}

int model_create_impl(uis_model** out, int device, int D, int H, int depth, const float* w_ih, const float* w_hh,
                      const float* b_ih, const float* b_hh, const float* w1, const float* b1, const float* w2,
                      const float* b2, const float* h0, const float* sigma2, double transition_bias, double crp_alpha,
                      int D_user, int H_user) {
  if (!(transition_bias > 0.0 && transition_bias < 1.0))
    return fail(UIS_ERR_INVALID, "transition_bias must be in (0,1), got %g", transition_bias);
  if (!(crp_alpha > 0.0)) return fail(UIS_ERR_INVALID, "crp_alpha must be > 0");
  uis::DeviceGuard device_guard_(device);
  CU(device_guard_.status);
  uis_model* m = new uis_model();
  m->device = device; m->D = D; m->H = H; m->depth = depth; m->p0 = transition_bias; m->alpha = crp_alpha;
  m->D_user = D_user; m->H_user = H_user;
  int rc = 0;
  auto body = [&]() -> int {
    cudaDeviceProp prop;
    CU(cudaGetDeviceProperties(&prop, device));
    m->num_sms = prop.multiProcessorCount;
    std::vector<float> v;
    // w_ih = [layer 0: 3H x D | layers >= 1: 3H x H each]; w_hh = depth x [3H x H]; b_ih, b_hh = depth x [3H]
    const size_t n_ih = (size_t)3 * H * D + (size_t)(depth - 1) * 3 * H * H;
    if (int r = fetch(v, w_ih, n_ih)) return r;
    {
      std::vector<float> l0(v.begin(), v.begin() + (size_t)3 * H * D);
      auto t = transpose(l0, 3 * H, D);
      if (int r = upload(m->wih_t, t.data(), t.size() * 4)) return r;
      std::vector<float> up;
      for (int l = 1; l < depth; ++l) {
        std::vector<float> w(v.begin() + (size_t)3 * H * D + (size_t)(l - 1) * 3 * H * H,
                             v.begin() + (size_t)3 * H * D + (size_t)l * 3 * H * H);
        auto tt = transpose(w, 3 * H, H);
        up.insert(up.end(), tt.begin(), tt.end());
      }
      if (up.empty()) up.resize(4, 0.f);
      if (int r = upload(m->wih_up_t, up.data(), up.size() * 4)) return r;
    }
    if (int r = fetch(v, w_hh, (size_t)depth * 3 * H * H)) return r;
    {
      std::vector<float> all;
      for (int l = 0; l < depth; ++l) {
        std::vector<float> w(v.begin() + (size_t)l * 3 * H * H, v.begin() + (size_t)(l + 1) * 3 * H * H);
        auto tt = transpose(w, 3 * H, H);
        all.insert(all.end(), tt.begin(), tt.end());
      }
      if (int r = upload(m->whh_t, all.data(), all.size() * 4)) return r;
    }
    if (int r = fetch(v, w1, (size_t)H * H)) return r;
    { auto t = transpose(v, H, H); if (int r = upload(m->w1_t, t.data(), t.size() * 4)) return r; }
    if (int r = fetch(v, w2, (size_t)D * H)) return r;
    { auto t = transpose(v, D, H); if (int r = upload(m->w2_t, t.data(), t.size() * 4)) return r; }
    if (int r = fetch(v, b_ih, (size_t)depth * 3 * H)) return r;
    if (int r = upload(m->bih, v.data(), v.size() * 4)) return r;
    if (int r = fetch(v, b_hh, (size_t)depth * 3 * H)) return r;
    if (int r = upload(m->bhh, v.data(), v.size() * 4)) return r;
    if (int r = fetch(v, b1, H)) return r;
    if (int r = upload(m->b1, v.data(), v.size() * 4)) return r;
    if (int r = fetch(v, b2, D)) return r;
    if (int r = upload(m->b2, v.data(), v.size() * 4)) return r;
    if (int r = fetch(v, sigma2, D)) return r;
    for (float& s : v) s = 1.0f / (2.0f * s);  // weight = 1 / (2 * sigma2), two fp32 ops (uisrnn.py:414)
    if (int r = upload(m->wvec, v.data(), v.size() * 4)) return r;
    std::vector<float> h0v;
    if (int r = fetch(h0v, h0, (size_t)depth * H)) return r;
    DevBuf h0d;
    if (int r = upload(h0d, h0v.data(), (size_t)depth * H * 4)) return r;
    if (int r = m->mean0.ensure(D * 4)) return r;
    if (int r = m->hidden0.ensure((size_t)depth * H * 4)) return r;
    uis::init_state_kernel<<<1, H, 3 * H * sizeof(float)>>>(m->whh_t.as<float>(), m->wih_up_t.as<float>(),
                                                           m->w1_t.as<float>(), m->w2_t.as<float>(),
                                                           m->bih.as<float>(), m->bhh.as<float>(), m->b1.as<float>(),
                                                           m->b2.as<float>(), h0d.as<float>(), H, D, depth,
                                                           m->mean0.as<float>(), m->hidden0.as<float>());
    CU(cudaGetLastError());
    CU(cudaDeviceSynchronize());
    h0d.release();
    if (depth == 1) {  // tensor-core pass: fp16 hi/lo planes of the untransposed (K-major) matrices + tensor map
      std::vector<float> whh0, w1v, b1v, w2v, hid0((size_t)H);
      if (int r = fetch(whh0, w_hh, (size_t)3 * H * H)) return r;
      if (int r = fetch(w1v, w1, (size_t)H * H)) return r;
      if (int r = fetch(b1v, b1, H)) return r;
      if (int r = fetch(w2v, w2, (size_t)D * H)) return r;
      CU(cudaMemcpy(hid0.data(), m->hidden0.p, (size_t)H * 4, cudaMemcpyDeviceToHost));
      if (int r = tc_prepare(m, whh0, w1v, b1v, w2v, hid0)) return r;
    }
    return 0;
  };
  rc = body();
  if (rc) {
    uis_model_destroy(m);
    return rc;
  }
  *out = m;
  return 0;
}

// ---- planning ----------------------------------------------------------------------------------------------------

// The decoding parameters of a call: `count` (crp_alpha, transition_bias) pairs.  A call without a sweep decodes the
// model's own pair.
struct DecodeParams {
  int count = 1;
  const double* alpha = nullptr;
  const double* p0 = nullptr;
};

DecodeParams model_decode(const uis_model* m) { return DecodeParams{1, &m->alpha, &m->p0}; }

// Rejects a sweep the kernels cannot run: no pairs, more than INT_MAX jobs, or a value out of range.
int check_decode(const uis_decode_params* dp, int U, DecodeParams* out) {
  if (!dp) return fail(UIS_ERR_INVALID, "decode_params is NULL");
  if (dp->count < 1) return fail(UIS_ERR_INVALID, "decode_params: count=%d (need >= 1)", dp->count);
  if (!dp->crp_alpha || !dp->transition_bias) return fail(UIS_ERR_INVALID, "decode_params: null value array");
  if ((long long)std::max(U, 1) * dp->count > std::numeric_limits<int>::max())
    return fail(UIS_ERR_INVALID, "decode_params: %d utterances x %d pairs exceeds INT_MAX jobs", U, dp->count);
  for (int c = 0; c < dp->count; ++c) {
    const double a = dp->crp_alpha[c], b = dp->transition_bias[c];
    if (!(std::isfinite(a) && a > 0.0))
      return fail(UIS_ERR_INVALID, "decode_params pair %d: crp_alpha=%g (need finite and > 0)", c, a);
    if (!(std::isfinite(b) && b > 0.0 && b < 1.0))
      return fail(UIS_ERR_INVALID, "decode_params pair %d: transition_bias=%g (need finite and in (0, 1))", c, b);
  }
  *out = DecodeParams{dp->count, dp->crp_alpha, dp->transition_bias};
  return 0;
}

struct Plan {
  int B, L, T, Kcap, ctas, P, maxN, G;
  uis::Kernel kernel = uis::Kernel::Beam;
  bool forced = false;  // the caller asked for this latency mode: a refused launch is an error, not a fallback
  int cluster = 1;      // Kernel::Cluster: CTAs per utterance (thread-block cluster size)
  int node_cap = 0, leaf_cap = 0, maxTN = 0, maxSteps = 0;  // look_ahead >= 2 only
  // look_ahead >= 2: the spill kernel that decodes, from a device-memory arena, what outgrew shared memory.  It runs
  // after Kernel::Tree, or instead of it as Kernel::TreeSpill (UISRNN_B200_TREE_SPILL=force); spill_ctas = 0: off.
  int spill_ctas = 0, spill_ni = 0, spill_nlf = 0, spill_P = 0;
  size_t spill_arena = 0, spill_budget = 0;  // arena bytes per spill CTA; the budget they were sized from
  long long rows;
};

// Pool slots held by a plan's CTAs: the shared-memory kernel's and the spill kernel's run one after the other on the
// same stream and share the pools.
size_t pool_slots(const Plan& pl) {
  return std::max((size_t)pl.ctas * pl.G * pl.P, (size_t)pl.spill_ctas * pl.spill_P);
}

// Sizes the spill kernel of a look-ahead plan.  The worst-case tree of one beam step at (B, Kcap, L) has
// B * sum_{i=1}^{L-1} prod_{j<i} (Kcap + 1 + j) interior nodes plus the B winners, and B * prod_{j<L} (Kcap + 1 + j)
// leaves.  Each spill CTA needs an arena for that tree and slot pools for its P; both are clipped (in proportion) to
// the byte budget: UISRNN_B200_TREE_SPILL_MB, else the smaller of 2 GiB and a quarter of the free device memory.
void plan_tree_spill(uis_model* m, Plan* pl) {
  if (const char* env = std::getenv("UISRNN_B200_TREE_SPILL")) {
    if (std::strcmp(env, "force") == 0) pl->kernel = uis::Kernel::TreeSpill;
    else if (env[0] == '0') return;
  }
  size_t budget;
  if (const char* env = std::getenv("UISRNN_B200_TREE_SPILL_MB")) {
    budget = (size_t)std::max(0ll, std::atoll(env)) << 20;
  } else {
    size_t free_b = 0, total_b = 0;
    uis::DeviceGuard g(m->device);
    if (g.status != cudaSuccess || cudaMemGetInfo(&free_b, &total_b) != cudaSuccess) { (void)cudaGetLastError(); free_b = 0; }
    budget = std::min<size_t>((size_t)2 << 30, (free_b + m->tree_arena.cap) / 4);  // the arena held is re-used
  }
  const int B = pl->B, K = pl->Kcap, L = pl->L;
  const double slot_bytes = 4.0 * (m->D + m->depth * m->H + 1);
  double ni = B, prod = 1;
  for (int i = 1; i < L; ++i) { prod *= K + i; ni += B * prod; }
  double nlf = B * prod * (K + L);
  auto cost = [&](double n, double l) {
    const int P = B * K + (int)n + B + 1;
    return (double)uis::make_tree_arena((int)n, (int)l, P).total + P * slot_bytes;
  };
  // leaf positions are stored in 32 bits, parent node indices in 24 (l_pc = parent << 8 | cluster)
  const double kMaxNi = (1 << 24) - 1, kMaxLeaves = 1 << 30;
  if (ni > kMaxNi) { nlf *= kMaxNi / ni; ni = kMaxNi; }
  if (nlf > kMaxLeaves) { ni *= kMaxLeaves / nlf; nlf = kMaxLeaves; }
  for (double f = std::min(1.0, (double)budget / cost(ni, nlf)); cost(ni, nlf) > (double)budget && ni > 64; f = 0.9) {
    ni = std::floor(ni * f);
    nlf = std::floor(nlf * f);
  }
  pl->spill_ni = std::max(64, (int)ni);  // floor: one CTA with about the smallest on-chip tree
  pl->spill_nlf = std::max(8 * 64, (int)nlf);
  pl->spill_P = B * K + pl->spill_ni + B + 1;
  const double per_cta = cost(pl->spill_ni, pl->spill_nlf);
  pl->spill_ctas = (int)std::max(1.0, std::min((double)pl->ctas, std::floor((double)budget / per_cta)));
  pl->spill_arena = uis::make_tree_arena(pl->spill_ni, pl->spill_nlf, pl->spill_P).total;
  pl->spill_budget = budget;
}

// U utterances (rows, frame counts) decoded as U * configs jobs (engine, lanes, CTAs and latency modes).
int make_plan(uis_model* m, const int64_t* off, int U, const uis_predict_opts* o, Plan* pl, int configs = 1) {
  if (!m || !o || (U > 0 && !off)) return fail(UIS_ERR_INVALID, "null argument");
  if (U < 0) return fail(UIS_ERR_INVALID, "U < 0");
  if (o->beam_size < 1 || o->look_ahead < 1 || o->test_iteration < 1)
    return fail(UIS_ERR_INVALID, "beam_size, look_ahead and test_iteration must be >= 1");
  if (o->look_ahead > 8) return fail(UIS_ERR_UNSUPPORTED, "look_ahead=%d > 8 not supported", o->look_ahead);
  if (o->beam_size > uis::kMaxBeam) return fail(UIS_ERR_UNSUPPORTED, "beam_size=%d > %d not supported", o->beam_size, uis::kMaxBeam);
  if (o->beam_size > 32 && o->look_ahead > 1)
    return fail(UIS_ERR_UNSUPPORTED, "beam_size=%d > 32 is supported with look_ahead 1 only (look_ahead=%d)", o->beam_size, o->look_ahead);
  if (o->engine < 0 || o->engine > 2) return fail(UIS_ERR_INVALID, "engine must be 0 (auto), 1 (FFMA) or 2 (tensor cores)");
  pl->B = o->beam_size;
  pl->L = o->look_ahead;
  pl->T = o->test_iteration;
  const bool tree = pl->L > 1;
  pl->Kcap = o->kcap > 0 ? o->kcap : (tree ? 16 : 32);
  if (o->kcap <= 0 && pl->B > 32)  // wide beams: the per-hypothesis tables (B * kcap entries) must fit shared memory
    while (pl->Kcap > 4 && kernel_smem(m, uis::Kernel::Beam, beam_sizes(pl->B, pl->Kcap, 1)) > uis::kSmemCap) pl->Kcap /= 2;
  if (pl->Kcap > (pl->B > 32 ? 511 : 2047) || pl->B * pl->Kcap + pl->B + 1 > 65535) return fail(UIS_ERR_INVALID, "kcap too large");
  if (tree && pl->Kcap > 255) return fail(UIS_ERR_UNSUPPORTED, "look_ahead >= 2 supports kcap <= 255");
  pl->P = pl->B * pl->Kcap + pl->B + 1;
  pl->rows = U > 0 ? off[U] : 0;
  int maxN = 0;
  for (int u = 0; u < U; ++u) {
    const long long n = off[u + 1] - off[u];
    if (n < 0) return fail(UIS_ERR_INVALID, "frame_offsets not monotone");
    if (n * pl->T > (1ll << 30)) return fail(UIS_ERR_INVALID, "utterance too long");
    maxN = std::max<long long>(maxN, n);
  }
  pl->maxN = std::max(maxN, 1);
  const long long J = (long long)U * configs;  // jobs
  int ctas = o->n_ctas > 0 ? o->n_ctas : m->num_sms;
  // lanes (utterances advanced together by one CTA, sharing each weight pass): 2 when there is
  // enough work to keep every CTA's lanes busy, else 1 (latency mode); opts->lanes overrides.
  int G = o->lanes > 0 ? std::min(o->lanes, 4) : (J >= 2ll * ctas ? 2 : 1);
  if (tree) {
    // look-ahead tree kernel: one utterance per CTA; size the on-chip node / leaf arrays to what
    // shared memory allows (internal nodes : leaves ~ 1 : 8, the typical fan-out K+2)
    G = 1;
    long long tn = 0;
    for (int u = 0; u < U; ++u) tn = std::max<long long>(tn, (off[u + 1] - off[u]) * pl->T);
    pl->maxTN = (int)std::max<long long>(tn, 1);
    pl->maxSteps = (pl->maxTN + pl->L - 1) / pl->L;
    int ni = 64;
    auto fits = [&](int n) {
      uis::BeamParams q = beam_sizes(pl->B, pl->Kcap, 1);
      q.L = pl->L; q.node_cap = n; q.leaf_cap = 8 * n; q.P = pl->B * pl->Kcap + n + pl->B + 1;
      return kernel_smem(m, uis::Kernel::Tree, q) <= uis::kSmemCap;
    };
    if (!fits(ni)) return fail(UIS_ERR_UNSUPPORTED, "look_ahead=%d beam_size=%d kcap=%d does not fit in shared memory", pl->L, pl->B, pl->Kcap);
    while (ni < 4096 && fits(ni + 32)) ni += 32;
    pl->node_cap = ni;
    pl->leaf_cap = 8 * ni;
    pl->P = pl->B * pl->Kcap + ni + pl->B + 1;
    pl->kernel = uis::Kernel::Tree;
  } else {
    // Tensor-core engine (look_ahead 1, depth 1, 128-row-tileable shapes): the cost of a weight pass does not depend on
    // the number of columns, so a CTA advances up to kTcColumns / 8 utterances together (a lane needs ~6 columns per step,
    // at most beam_size + 1).  Chosen automatically when some CTA gets more than one utterance; below that the
    // one-lane FFMA kernel or the cluster (latency) mode is faster.  Its device tables default to 16 clusters per
    // hypothesis (UIS_ERR_OVERFLOW asks the caller for more, as always).
    if (o->engine != 1 && m->tc_ready && o->cluster <= 0) {
      const int kc = o->kcap > 0 ? o->kcap : 16;
      auto tc_smem = [&](int g) { return kernel_smem(m, uis::Kernel::TensorCore, beam_sizes(pl->B, kc, g)); };
      if (tc_smem(1) != uis::kNoKernel) {
        int Gt = o->lanes > 0 ? std::min(o->lanes, (int)uis::kMaxLanes)
                              : (int)std::min<long long>(uis::kTcColumns / 8, (J + ctas - 1) / std::max(ctas, 1));
        Gt = std::max(Gt, 1);
        while (Gt > 1 && (tc_smem(Gt) > uis::kSmemCap || Gt * pl->B > 256)) --Gt;
        const bool fits = tc_smem(Gt) <= uis::kSmemCap && pl->B * kc + pl->B + 1 <= 65535;
        if (fits && (o->engine == 2 || J > ctas)) {
          pl->kernel = uis::Kernel::TensorCore;
          pl->Kcap = kc;
          pl->P = pl->B * kc + pl->B + 1;
          G = Gt;
        } else if (o->engine == 2) {
          return fail(UIS_ERR_UNSUPPORTED, "tensor-core engine: beam_size=%d kcap=%d does not fit in shared memory", pl->B, kc);
        }
      } else if (o->engine == 2) {
        return fail(UIS_ERR_UNSUPPORTED, "tensor-core engine: no kernel for hidden=%d dim=%d", m->H, m->D);
      }
    } else if (o->engine == 2) {
      return fail(UIS_ERR_UNSUPPORTED, "tensor-core engine needs look_ahead 1, depth 1, hidden/dim multiples of 128, no "
                                       "cluster mode and weights its fp16 split holds (uis_model_create)");
    }
    if (pl->kernel != uis::Kernel::TensorCore)
      while (G > 1 && kernel_smem(m, uis::Kernel::Beam, beam_sizes(pl->B, pl->Kcap, G)) > uis::kSmemCap) --G;
    while (G > 1 && G * pl->B > 256) --G;  // at most 256 (lane, winner) pairs per CTA step
  }
  if (tree && o->engine == 2) return fail(UIS_ERR_UNSUPPORTED, "tensor-core engine: look_ahead must be 1");
  pl->G = G;
  pl->ctas = (int)std::max(1ll, std::min<long long>(ctas, std::max((J + G - 1) / G, 1ll)));
  if (tree) plan_tree_spill(m, pl);
  // Cluster (latency) mode: with fewer utterances than SMs, a thread-block cluster of 2/4/8 CTAs works on
  // each utterance (k-split of every weight matrix, uis_beam.cuh).  opts->cluster: 0 = auto (largest of 4, 2
  // that still gives every utterance its own cluster), -1 = off, 2/4/8 = forced.
  // Stationary-weights mode (uis_beam_stat.cuh): 32 CTAs per utterance keep the weights in shared memory.  The fastest
  // way to decode up to #SMs / 32 utterances at a time; opts->cluster = 32 forces it, 0 picks it automatically.
  if (!tree && U >= 1 && (o->cluster == 0 || o->cluster == uis::kStatGroup) && m->depth == 1 &&
      o->lanes <= 1 && o->engine != 2) {
    const bool want = o->cluster == uis::kStatGroup || (J * uis::kStatGroup <= ctas && o->engine == 0 && o->n_ctas <= 0);
    const int kc = o->kcap > 0 ? o->kcap : 32;
    const bool can = ctas >= uis::kStatGroup && kernel_smem(m, uis::Kernel::Stat, beam_sizes(pl->B, kc, 1)) <= uis::kSmemCap &&
                     pl->B * kc + pl->B + 1 <= 65535;
    if (want && can) {
      const int groups = (int)std::max(1ll, std::min<long long>(ctas / uis::kStatGroup, J));
      pl->kernel = uis::Kernel::Stat;
      pl->forced = o->cluster == uis::kStatGroup;
      pl->Kcap = kc;
      pl->P = pl->B * kc + pl->B + 1;
      pl->G = 1;
      pl->ctas = groups * uis::kStatGroup;
      return 0;
    }
    if (o->cluster == uis::kStatGroup)
      return fail(UIS_ERR_UNSUPPORTED, "stationary-weights mode needs hidden=512 dim=256 depth=1, >= 32 CTAs and beam_size/kcap that fit in shared memory");
  }
  if (pl->kernel == uis::Kernel::Beam && U >= 1 && o->cluster >= 0 && m->depth == 1 && o->lanes <= 1) {
    int cs = 0;
    if (o->cluster == 2 || o->cluster == 4 || o->cluster == 8) {
      cs = o->cluster;
    } else if (o->cluster == 0) {
      for (int c : {4, 2})
        if (J * c <= ctas) { cs = c; break; }
    } else {
      return fail(UIS_ERR_INVALID, "cluster must be -1, 0, 2, 4, 8 or 32");
    }
    if (cs > 1 && kernel_smem(m, uis::Kernel::Cluster, beam_sizes(pl->B, pl->Kcap, 1)) <= uis::kSmemCap) {
      const int clusters = (int)std::max(1ll, std::min<long long>(ctas / cs, J));
      pl->kernel = uis::Kernel::Cluster;
      pl->cluster = cs;
      pl->forced = o->cluster > 0;
      pl->G = 1;
      pl->ctas = clusters * cs;
    } else if (o->cluster > 0) {
      return fail(UIS_ERR_UNSUPPORTED, "cluster mode needs hidden=512 dim=256 depth=1 and beam_size/kcap that fit in shared memory");
    }
  }
  return 0;
}

size_t workspace_bytes(const uis_model* m, const Plan& pl, int U, int configs = 1) {
  const size_t J = (size_t)U * configs;
  size_t b = 0;
  b += (size_t)pl.rows * 3 * m->H * 4;                                  // gi
  b += pool_slots(pl) * (m->D + m->depth * m->H + 1) * 4;            // slot pools (+ Gaussian term per slot)
  b += (size_t)pl.spill_ctas * pl.spill_arena;                          // look-ahead spill arenas
  b += (size_t)pl.ctas * pl.G * (pl.L > 1 ? (size_t)pl.maxTN + pl.maxSteps : (size_t)pl.maxN) * pl.B * 4;  // back-pointers
  b += (size_t)(U + 1) * 8 + J * 8 + 256;                               // offsets, order, status
  if (configs > 1) b += (size_t)configs * (4096 + 3) * 8;               // log tables of the sweep (at least)
  if (pl.kernel == uis::Kernel::TensorCore)                             // a = relu(W1 h' + b1) between two products
    b += (size_t)pl.ctas * uis::kTcColumns * m->H * 4;
  return b;
}

// ---- groups: lists larger than the device, decoded or scored in groups of whole utterances ---------------------
//
// Utterances are independent in every beam and score kernel (uisrnn.py:587-589), and a score chain never crosses an
// utterance, so a list whose per-frame workspace does not fit the device runs as consecutive groups of whole
// utterances, one after the other on the call's stream, each planned on its own.  Every entry point decides the
// group size here.

// Frames one group may hold: UISRNN_B200_MAX_ROWS when set (>= 1), else what fits in 90% of the free device memory plus
// the `held` bytes of handle buffers that the call re-uses, after `fixed` bytes that do not grow with the frames, at
// `per_row` bytes per frame.  At least 1.
int row_budget(size_t per_row, size_t fixed, size_t held, size_t* max_rows) {
  if (const char* env = std::getenv("UISRNN_B200_MAX_ROWS")) {
    *max_rows = (size_t)std::max(1ll, std::atoll(env));
    return 0;
  }
  size_t free_b = 0, total_b = 0;
  CU(cudaMemGetInfo(&free_b, &total_b));
  const double budget = 0.9 * (double)(free_b + held) - (double)fixed;
  *max_rows = budget > (double)per_row ? (size_t)(budget / (double)per_row) : 1;
  return 0;
}

// Group boundaries of U utterances (frame offsets `off`) under a budget of max_rows frames: {0, u1, ..., U}, each group
// as many consecutive whole utterances as fit, an utterance longer than max_rows a group of its own.
std::vector<int> cut_groups(const int64_t* off, int U, size_t max_rows) {
  std::vector<int> cuts{0};
  for (int u0 = 0; u0 < U;) {
    int u1 = u0 + 1;
    while (u1 < U && (size_t)(off[u1 + 1] - off[u0]) <= max_rows) ++u1;
    cuts.push_back(u1);
    u0 = u1;
  }
  if (U == 0) cuts.push_back(0);  // an empty list: one empty group
  return cuts;
}

// Frame offsets of utterances [u0, u1), rebased to the group's first row.
std::vector<int64_t> group_offsets(const int64_t* off, int u0, int u1) {
  std::vector<int64_t> g(u1 - u0 + 1);
  for (int q = u0; q <= u1; ++q) g[q - u0] = off[q] - off[u0];
  return g;
}

// Where one group of a call run in groups sits in the whole call (the defaults: a call of one group).
struct Group {
  int index = 0;         // groups of the call that launched kernels before this one: the first resets the device
                         // counters and uses events 0..2, the later ones add to the counters and use their own events
  int job0 = 0;          // the group's first job in the call's per-job status
  long long plane = 0;   // the call's rows: the row stride of its label planes and per-frame score outputs (0: the group's)
  int stride = 0;        // the call's U: the row stride of its [configs][U] score totals (0: the group's)
};

// Bytes of the queue counters at the head of queue_stats: a later group resets only these, so that the device
// counters behind them add up over the groups of a call.
constexpr size_t kQueueBytes = 8 * sizeof(unsigned long long);

// Adds the stats of one group to those of the groups before it.
void add_stats(uis_stats* a, const uis_stats& b) {
  a->utterances += b.utterances; a->frames += b.frames; a->beam_steps += b.beam_steps; a->gru_columns += b.gru_columns;
  a->weight_passes += b.weight_passes; a->candidates += b.candidates; a->kernel_launches += b.kernel_launches;
  a->ctas = std::max(a->ctas, b.ctas); a->max_k = std::max(a->max_k, b.max_k);
  a->prepass_ms += b.prepass_ms; a->beam_ms += b.beam_ms; a->h2d_ms += b.h2d_ms; a->pipeline_ms += b.pipeline_ms;
  a->lanes = std::max(a->lanes, b.lanes); a->cluster = std::max(a->cluster, b.cluster);
  a->engine = std::max(a->engine, b.engine); a->tc_columns = std::max(a->tc_columns, b.tc_columns);
  for (int i = 0; i < 10; ++i) a->phase_cycles[i] += b.phase_cycles[i];
  for (int i = 0; i < 4; ++i) a->tc_cycles[i] += b.tc_cycles[i];
  a->chunks += b.chunks; a->groups += b.groups; a->staged = std::max(a->staged, b.staged);
}

// Creates the three events of group g.
int group_events(uis_model* m, int g) {
  if (m->ev.size() < (size_t)3 * (g + 1)) m->ev.resize((size_t)3 * (g + 1), nullptr);
  for (auto& e : m->ev)
    if (!e) CU(cudaEventCreate(&e));
  return 0;
}

// Speaker bounds of a bounded call (host arrays, either may be NULL): 0 = no bound, max >= 1, 0 <= min <= max.
struct SpeakerBounds {
  const int32_t* max = nullptr;
  const int32_t* min = nullptr;
  int32_t* out_dev = nullptr;  // [U] device, may be NULL
  SpeakerBounds at(int u0) const {
    return SpeakerBounds{max ? max + u0 : nullptr, min ? min + u0 : nullptr, out_dev ? out_dev + u0 : nullptr};
  }
};

// N-best outputs of a call (n_best = 1 with NULL pointers: a plain call).  Labels are n_best planes of the call's rows.
struct NBestOut {
  int k = 1;
  float* scores = nullptr;     // [U][k]
  int32_t* speakers = nullptr; // [U][k]
  int32_t* count = nullptr;    // [U]
};

int check_bounds(int U, const int32_t* mx, const int32_t* mn) {
  for (int u = 0; u < U; ++u) {
    const int a = mx ? mx[u] : 0, b = mn ? mn[u] : 0;
    if (a < 0 || b < 0 || (a > 0 && b > a))
      return fail(UIS_ERR_INVALID, "utterance %d: max_speakers=%d min_speakers=%d (need max >= 1 or 0 = none, "
                  "min >= 0, min <= max)", u, a, b);
  }
  return 0;
}

// n_best in [1, beam_size]; an N-best call needs its label and score buffers.
int check_nbest(int n_best, const uis_predict_opts* opts, const uis_nbest_out* out) {
  if (n_best < 1 || n_best > opts->beam_size)
    return fail(UIS_ERR_INVALID, "n_best=%d (need 1 <= n_best <= beam_size=%d)", n_best, opts->beam_size);
  if (!out->scores) return fail(UIS_ERR_INVALID, "n_best: null scores buffer");
  return 0;
}

// ---- launch ------------------------------------------------------------------------------------------------------

// What launch errors call each uis::Kernel: the missing instantiation, the kernel.
const struct { const char *missing, *name; } kKernelNames[] = {
    {"sm_90a kernel instantiated", "beam kernel"},
    {"cluster-mode kernel", "cluster beam kernel"},
    {"stationary-weights kernel", "stationary-weights beam kernel"},
    {"tensor-core kernel", "tensor-core beam kernel"},
    {"sm_90a kernel instantiated", "look-ahead kernel"},
    {"sm_90a kernel instantiated", "look-ahead kernel"},
};

// Launches kernel k of plan `pl` on `ctas` CTAs and records its CTAs per utterance in stats.cluster.  A latency mode
// that the planner chose on its own and whose launch is refused (e.g. a partitioned GPU that cannot co-schedule the
// CTAs) gives way to the FFMA kernel on the same grid: its extra CTAs find the utterance queue empty.
int launch(uis_model* m, const Plan& pl, uis::Kernel k, const uis::BeamParams& p, int ctas, cudaStream_t st) {
  using uis::Kernel;
  const unsigned smem = kernel_smem(m, k, p);
  if (smem > uis::kSmemCap) {
    if (k == Kernel::Tree || k == Kernel::TreeSpill)
      return fail(UIS_ERR_UNSUPPORTED, "look_ahead=%d beam_size=%d kcap=%d needs %u B of shared memory (> 227 KB)", p.L,
                  p.B, p.Kcap, smem);
    return fail(UIS_ERR_UNSUPPORTED, "beam_size=%d kcap=%d lanes=%d needs %u B of shared memory (> 227 KB); lower kcap",
                p.B, p.Kcap, p.G, smem);
  }
  cudaError_t e = cudaSuccess;
  const bool have = launch_kernel(m, k, p, ctas, pl.cluster, smem, st, &e);
  if (have && e == cudaSuccess) {
    m->stats.cluster = k == Kernel::Stat ? uis::kStatGroup : k == Kernel::Cluster ? pl.cluster : 1;
    return 0;
  }
  if ((k == Kernel::Cluster || k == Kernel::Stat) && !pl.forced) {
    (void)cudaGetLastError();  // clear the launch error and fall back
    return launch(m, pl, Kernel::Beam, p, ctas, st);
  }
  if (!have)
    return fail(UIS_ERR_UNSUPPORTED, "no %s for hidden=%d dim=%d", kKernelNames[(int)k].missing, m->H, m->D);
  return fail(UIS_ERR_CUDA, "%s launch failed: %s", kKernelNames[(int)k].name, cudaGetErrorString(e));
}

// ---- run_device --------------------------------------------------------------------------------------------------

// Log tables for decodes of up to max_tn frames under `dp`, built on the host with std::log so that a config's values
// are those a model created with its pair uses.  Fills the table pointers of `p`.
int ensure_log_tables(uis_model* m, int max_tn, const DecodeParams& dp, uis::BeamParams* p) {
  const int need = max_tn + 2;
  if (need > m->log_cap) {
    const int cap = std::max(need, 4096);
    std::vector<double> ln(cap);
    ln[0] = -INFINITY;
    for (int i = 1; i < cap; ++i) ln[i] = std::log((double)i);  // np.log(block_counts[c])
    if (int rc = upload(m->logn, ln.data(), cap * sizeof(double))) return rc;
    m->log_cap = cap;
  }
  // the model's own pair (by value: the Python binding passes it as a one-pair sweep) keeps its own tables, so that
  // alternating plain calls with a sweep does not rebuild a table on every call
  const bool own = dp.count == 1 && std::memcmp(dp.alpha, &m->alpha, sizeof(double)) == 0 &&
                   std::memcmp(dp.p0, &m->p0, sizeof(double)) == 0;
  uis_model::LogTables& t = own ? m->own_logs : m->sweep_logs;
  std::vector<double> key;
  for (int c = 0; c < dp.count; ++c) { key.push_back(dp.alpha[c]); key.push_back(dp.p0[c]); }
  if (need > t.cap || key != t.key) {
    const int cap = std::max({need, 4096, t.cap});
    if (t.cap) CU(cudaDeviceSynchronize());  // the tables are rewritten in place: no earlier call may still read them
    std::vector<double> lt((size_t)dp.count * cap), cv((size_t)dp.count * 3);
    for (int c = 0; c < dp.count; ++c) {
      for (int i = 0; i < cap; ++i) lt[(size_t)c * cap + i] = std::log((double)i + dp.alpha[c]);  // np.log(sum(block_counts) + alpha)
      cv[3 * c] = std::log(dp.p0[c]);            // np.log(self.transition_bias)      uisrnn.py:418
      cv[3 * c + 1] = std::log(1.0 - dp.p0[c]);  // np.log(1 - self.transition_bias)  uisrnn.py:416
      cv[3 * c + 2] = std::log(dp.alpha[c]);     // np.log(self.crp_alpha)            uisrnn.py:445
    }
    t.cap = 0;
    t.key.clear();
    if (int rc = upload(t.tot, lt.data(), lt.size() * sizeof(double))) return rc;
    if (int rc = upload(t.cfg, cv.data(), cv.size() * sizeof(double))) return rc;
    t.cap = cap;
    t.key = key;
  }
  p->logn = m->logn.as<double>();
  p->logtot = t.tot.as<double>();
  p->cfg_log = t.cfg.as<double>();
  p->logtot_stride = t.cap;
  return 0;
}

// The model's part of the kernel parameters: weights and constants (ensure_log_tables adds the log terms).
uis::BeamParams model_params(const uis_model* m) {
  const int H = m->H;
  uis::BeamParams p{};
  p.whh_t = m->whh_t.as<float>(); p.w1_t = m->w1_t.as<float>(); p.w2_t = m->w2_t.as<float>();
  p.depth = m->depth;
  for (int l = 1; l < m->depth; ++l) {
    p.wih_up_t[l - 1] = m->wih_up_t.as<float>() + (size_t)(l - 1) * H * 3 * H;
    p.whh_up_t[l - 1] = m->whh_t.as<float>() + (size_t)l * H * 3 * H;
  }
  p.bih_up = m->bih.as<float>() + 3 * H;   // layers >= 1
  p.bhh_up = m->bhh.as<float>() + 3 * H;
  p.bhh = m->bhh.as<float>(); p.b1 = m->b1.as<float>(); p.b2 = m->b2.as<float>();
  p.wvec = m->wvec.as<float>(); p.mean0 = m->mean0.as<float>(); p.hidden0 = m->hidden0.as<float>();
  return p;
}

// Decodes U utterances under dp.count configs: J = U * dp.count jobs, job j = utterance j % U under config j / U.
// Per-job outputs (status, N-best scores / speakers / counts, taps) are [J]; labels_dev holds dp.count * nb.k planes
// of the call's rows (plane c * nb.k + j: config c, hypothesis j), grp.plane rows apart when this is one group of a
// larger call.
int run_device(uis_model* m, const float* x_dev, const int64_t* off, int U, const Plan& pl, int32_t* labels_dev,
               const uis_debug_taps* taps, cudaStream_t st, const SpeakerBounds& sb, const NBestOut& nb,
               const DecodeParams& dp, bool gi_ready = false, const Group& grp = Group{}) {
  const int H = m->H, D = m->D;
  const int J = U * dp.count;
  if (sb.out_dev && U > 0) CU(cudaMemsetAsync(sb.out_dev, 0, (size_t)J * sizeof(int32_t), st));  // empty inputs: 0
  if (U > 0 && pl.rows == 0) {  // no kernel runs: every utterance is empty and returns no hypothesis
    if (nb.count) CU(cudaMemsetAsync(nb.count, 0, (size_t)J * sizeof(int32_t), st));
    if (nb.speakers) CU(cudaMemsetAsync(nb.speakers, 0, (size_t)J * nb.k * sizeof(int32_t), st));
    if (nb.scores) {
      const std::vector<float> inf((size_t)J * nb.k, std::numeric_limits<float>::infinity());
      CU(cudaMemcpyAsync(nb.scores, inf.data(), inf.size() * sizeof(float), cudaMemcpyHostToDevice, st));
      CU(cudaStreamSynchronize(st));  // (inf is about to go out of scope)
    }
  }
  m->stats = uis_stats{};
  m->stats.utterances = J;
  m->stats.frames = pl.rows;
  m->stats.ctas = pl.ctas;
  m->stats.lanes = pl.G;
  m->stats.cluster = pl.cluster;
  m->stats.groups = 1;
  m->last_U = J;
  m->last_groups = 1;
  m->last_score = false;
  m->last_tree_spill = pl.spill_ctas > 0;
  m->last_spill_ni = pl.spill_ni; m->last_spill_nlf = pl.spill_nlf; m->last_spill_budget = pl.spill_budget;
  m->last_stream = st;
  m->stats_pending = false;
  if (U == 0 || pl.rows == 0) {
    return 0;
  }
  uis::BeamParams p = model_params(m);
  long long max_tn = 0;
  for (int u = 0; u < U; ++u) max_tn = std::max<long long>(max_tn, (off[u + 1] - off[u]) * pl.T);
  if (int rc = ensure_log_tables(m, (int)max_tn, dp, &p)) return rc;

  // schedule: longest utterance first (LPT) -- steps are strictly sequential per utterance.  The configs of one
  // utterance follow each other, so that they read the same input rows at about the same time.
  std::vector<int> by_len(U), order((size_t)J);
  std::iota(by_len.begin(), by_len.end(), 0);
  std::stable_sort(by_len.begin(), by_len.end(),
                   [&](int a, int b) { return off[a + 1] - off[a] > off[b + 1] - off[b]; });
  for (int i = 0; i < U; ++i)
    for (int c = 0; c < dp.count; ++c) order[(size_t)i * dp.count + c] = c * U + by_len[i];
  std::vector<long long> off_ll(off, off + U + 1);

  if (int rc = m->row_off.ensure((U + 1) * sizeof(long long))) return rc;
  if (int rc = m->order.ensure((size_t)J * sizeof(int))) return rc;
  if (int rc = m->status.ensure((size_t)(grp.job0 + J) * sizeof(int))) return rc;
  if (int rc = m->queue_stats.ensure(40 * sizeof(unsigned long long))) return rc;
  if (int rc = m->gi.ensure((size_t)pl.rows * 3 * H * sizeof(float))) return rc;
  if (int rc = m->pool_mean.ensure(pool_slots(pl) * D * sizeof(float))) return rc;
  if (int rc = m->pool_hidden.ensure(pool_slots(pl) * m->depth * H * sizeof(float))) return rc;
  if (int rc = m->pool_mse.ensure(pool_slots(pl) * sizeof(float))) return rc;
  if (int rc = m->tree_arena.ensure((size_t)pl.spill_ctas * pl.spill_arena)) return rc;
  if (int rc = m->bp.ensure((size_t)pl.ctas * pl.G * (pl.L > 1 ? (size_t)pl.maxTN + pl.maxSteps : (size_t)pl.maxN) * pl.B *
                            sizeof(unsigned)))
    return rc;

  const bool tc = pl.kernel == uis::Kernel::TensorCore;
  if (tc)
    if (int rc = m->tc_scratch.ensure((size_t)pl.ctas * uis::kTcColumns * H * sizeof(float))) return rc;
  if (pl.kernel == uis::Kernel::Stat) {  // pl.ctas / kStatGroup groups
    if (int rc = m->stat_bar.ensure((size_t)pl.ctas * sizeof(unsigned))) return rc;
    if (int rc = m->stat_scratch.ensure((size_t)(pl.ctas / uis::kStatGroup) * uis::kCPCluster * H * sizeof(float))) return rc;
    CU(cudaMemsetAsync(m->stat_bar.p, 0, (size_t)pl.ctas * sizeof(unsigned), st));
  }

  CU(cudaMemcpyAsync(m->row_off.p, off_ll.data(), (U + 1) * sizeof(long long), cudaMemcpyHostToDevice, st));
  CU(cudaMemcpyAsync(m->order.p, order.data(), (size_t)J * sizeof(int), cudaMemcpyHostToDevice, st));
  CU(cudaMemsetAsync(m->queue_stats.p, 0, grp.index ? kQueueBytes : 40 * sizeof(unsigned long long), st));
  CU(cudaMemsetAsync(m->status.as<int>() + grp.job0, 0xff, (size_t)J * sizeof(int), st));

  p.x = x_dev; p.gi = m->gi.as<float>();
  p.row_off = m->row_off.as<long long>(); p.order = m->order.as<int>();
  p.U = J; p.n_utt = U; p.B = pl.B; p.Kcap = pl.Kcap; p.T = pl.T; p.P = pl.P; p.maxN = pl.maxN; p.G = pl.G;
  p.L = pl.L; p.node_cap = pl.node_cap; p.leaf_cap = pl.leaf_cap; p.maxTN = pl.maxTN; p.maxSteps = pl.maxSteps;
  p.pool_mean = m->pool_mean.as<float>(); p.pool_hidden = m->pool_hidden.as<float>(); p.pool_mse = m->pool_mse.as<float>();
  p.bp = m->bp.as<unsigned>();
  p.queue = m->queue_stats.as<int>();
  p.stats = m->queue_stats.as<unsigned long long>() + 8;
  p.labels = labels_dev; p.status = m->status.as<int>() + grp.job0;
  if (sb.max || sb.min) {
    std::vector<int32_t> kb(2 * (size_t)U);
    for (int u = 0; u < U; ++u) { kb[2 * u] = sb.max ? sb.max[u] : 0; kb[2 * u + 1] = sb.min ? sb.min[u] : 0; }
    if (int rc = m->spk_bound.ensure(kb.size() * sizeof(int32_t))) return rc;
    CU(cudaMemcpyAsync(m->spk_bound.p, kb.data(), kb.size() * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    p.spk_bound = m->spk_bound.as<int>();
  }
  p.spk_out = sb.out_dev;
  p.n_best = nb.k; p.label_plane = grp.plane ? grp.plane : pl.rows;
  p.nbest_scores = nb.scores; p.nbest_speakers = nb.speakers; p.nbest_count = nb.count;
  p.trace_utt = -1;
  if (pl.kernel == uis::Kernel::Stat) {
    p.stat_bar = m->stat_bar.as<unsigned>();
    p.stat_scratch = m->stat_scratch.as<float>();
  }
  if (tc) {
    p.tc_wmap = m->tc_map;
    p.tc_sh = m->tc_sh; p.tc_sa = m->tc_sa;
    p.tc_inv_hh = m->tc_inv_hh; p.tc_inv_1 = m->tc_inv_1; p.tc_inv_2 = m->tc_inv_2;
    p.tc_scratch = m->tc_scratch.as<float>();
  }

  long long trace_steps = 0;
  if (taps) {
    if (taps->final_scores) {
      if (int rc = m->dbg_final_scores.ensure((size_t)J * pl.B * 4)) return rc;
      p.dbg_final_scores = m->dbg_final_scores.as<float>();
      if (int rc = m->dbg_final_k.ensure((size_t)J * 4)) return rc;
      p.dbg_final_k = m->dbg_final_k.as<int>();
    }
    if (taps->trace_utt >= 0 && taps->trace_utt < J) {  // a job: utterance trace_utt % U under config trace_utt / U
      p.trace_utt = taps->trace_utt;
      p.trace_capacity = std::max(taps->trace_capacity, 0);
      const int tu = p.trace_utt % U;
      trace_steps = ((off[tu + 1] - off[tu]) * pl.T + pl.L - 1) / pl.L;
      if (taps->step_winners && p.trace_capacity > 0) {
        if (int rc = m->dbg_win.ensure((size_t)p.trace_capacity * 4 * (1 + pl.L))) return rc;
        if (int rc = m->dbg_score.ensure((size_t)p.trace_capacity * 4)) return rc;
        if (int rc = m->dbg_off.ensure((size_t)(trace_steps + 1) * 8)) return rc;
        p.dbg_win = m->dbg_win.as<int>(); p.dbg_score = m->dbg_score.as<float>();
        p.dbg_off = m->dbg_off.as<long long>();
      }
      if (taps->best_mean) {
        if (int rc = m->dbg_best_mean.ensure((size_t)pl.Kcap * D * 4)) return rc;
        if (int rc = m->dbg_best_hidden.ensure((size_t)pl.Kcap * m->depth * H * 4)) return rc;
        if (int rc = m->dbg_best_blocks.ensure((size_t)pl.Kcap * 4)) return rc;
        p.dbg_best_mean = m->dbg_best_mean.as<float>(); p.dbg_best_hidden = m->dbg_best_hidden.as<float>();
        p.dbg_best_blocks = m->dbg_best_blocks.as<int>();
      }
    }
  }

  if (int rc = group_events(m, grp.index)) return rc;
  cudaEvent_t* ev = m->ev.data() + 3 * grp.index;
  CU(cudaEventRecord(ev[0], st));
  // kernel 1: input projection GEMM (the host-buffer path has already run it chunk by chunk, under the H2D copies)
  if (!gi_ready) {
    dim3 grid((3 * H + uis::PBN - 1) / uis::PBN, (unsigned)((pl.rows + uis::PBM - 1) / uis::PBM));
    uis::input_proj_kernel<<<grid, 256, 0, st>>>(x_dev, m->wih_t.as<float>(), m->bih.as<float>(), m->gi.as<float>(),
                                                (int)pl.rows, 3 * H, D);
    CU(cudaGetLastError());
  }
  CU(cudaEventRecord(ev[1], st));
  // kernel 2: the planned persistent beam search.  Look-ahead: the spill kernel right behind it on the same stream
  // decodes the utterances it left at status -5 (every one under Kernel::TreeSpill) from a second queue; its CTAs find
  // nothing to do and exit when every tree fitted.
  if (pl.kernel != uis::Kernel::TreeSpill)
    if (int rc = launch(m, pl, pl.kernel, p, pl.ctas, st)) return rc;
  if (pl.spill_ctas) {
    uis::BeamParams ps = p;
    ps.node_cap = pl.spill_ni; ps.leaf_cap = pl.spill_nlf; ps.P = pl.spill_P;
    ps.queue = p.queue + 1;
    ps.tree_arena = m->tree_arena.as<unsigned char>();
    ps.tree_spill_all = pl.kernel == uis::Kernel::TreeSpill;
    if (int rc = launch(m, pl, uis::Kernel::TreeSpill, ps, pl.spill_ctas, st)) return rc;
  }
  m->stats.engine = tc ? 2 : 1;
  m->stats.tc_columns = tc ? uis::kTcColumns : 0;
  CU(cudaEventRecord(ev[2], st));
  m->stats.kernel_launches = 2 + (pl.kernel == uis::Kernel::Tree && pl.spill_ctas ? 1 : 0);
  m->stats_pending = true;

  if (taps) {
    CU(cudaStreamSynchronize(st));
    if (p.dbg_final_scores) {
      CU(cudaMemcpy(taps->final_scores, p.dbg_final_scores, (size_t)J * pl.B * 4, cudaMemcpyDeviceToHost));
      if (taps->final_k) CU(cudaMemcpy(taps->final_k, p.dbg_final_k, (size_t)J * 4, cudaMemcpyDeviceToHost));
    }
    if (p.dbg_win) {
      CU(cudaMemcpy(taps->step_winners, p.dbg_win, (size_t)p.trace_capacity * 4 * (1 + pl.L), cudaMemcpyDeviceToHost));
      CU(cudaMemcpy(taps->step_scores, p.dbg_score, (size_t)p.trace_capacity * 4, cudaMemcpyDeviceToHost));
      if (taps->step_offsets)
        CU(cudaMemcpy(taps->step_offsets, p.dbg_off, (size_t)(trace_steps + 1) * 8, cudaMemcpyDeviceToHost));
    }
    if (p.dbg_best_mean) {
      CU(cudaMemcpy2D(taps->best_mean, (size_t)m->D_user * 4, p.dbg_best_mean, (size_t)D * 4, (size_t)m->D_user * 4, pl.Kcap,
                      cudaMemcpyDeviceToHost));
      if (taps->best_hidden)
        CU(cudaMemcpy2D(taps->best_hidden, (size_t)m->H_user * 4, p.dbg_best_hidden, (size_t)H * 4, (size_t)m->H_user * 4,
                        (size_t)pl.Kcap * m->depth, cudaMemcpyDeviceToHost));
      if (taps->best_blocks)
        CU(cudaMemcpy(taps->best_blocks, p.dbg_best_blocks, (size_t)pl.Kcap * 4, cudaMemcpyDeviceToHost));
    }
  }
  return 0;
}

// prepass_ms and beam_ms of the last call: the sums over its groups' events.
int event_times(uis_model* m) {
  m->stats.prepass_ms = m->stats.beam_ms = 0.f;
  for (int g = 0; g < m->last_groups; ++g) {
    const cudaEvent_t* ev = m->ev.data() + 3 * g;
    float a = 0.f, b = 0.f;
    CU(cudaEventElapsedTime(&a, ev[0], ev[1]));
    CU(cudaEventElapsedTime(&b, ev[1], ev[2]));
    m->stats.prepass_ms += a;
    m->stats.beam_ms += b;
  }
  return 0;
}

// Pull the device-side counters and per-utterance status of the last call (synchronises).
int collect(uis_model* m) {
  if (!m->stats_pending) return 0;
  CU(cudaStreamSynchronize(m->last_stream));
  unsigned long long s[24];
  CU(cudaMemcpy(s, m->queue_stats.as<unsigned long long>() + 8, sizeof s, cudaMemcpyDeviceToHost));
  if (m->last_score) {  // the chain kernel's columns and passes; max_k came from the labels (or the device plans)
    m->stats.gru_columns = (int64_t)s[0];
    m->stats.weight_passes = (int64_t)s[1];
    if (m->last_score_counts) {  // {chains, queued, max_k, -} of every group
      std::vector<int> counts((size_t)4 * m->last_groups);
      CU(cudaMemcpy(counts.data(), m->sc_counts.p, counts.size() * sizeof(int), cudaMemcpyDeviceToHost));
      m->stats.max_k = 0;
      for (int g = 0; g < m->last_groups; ++g) m->stats.max_k = std::max(m->stats.max_k, counts[(size_t)4 * g + 2]);
    }
    if (int rc = event_times(m)) return rc;
    m->stats_pending = false;
    return 0;
  }
  for (int i = 0; i < 10; ++i) m->stats.phase_cycles[i] = (int64_t)s[8 + i];
  for (int i = 0; i < 4; ++i) m->stats.tc_cycles[i] = (int64_t)s[18 + i];
  m->stats.gru_columns = (int64_t)s[0];
  m->stats.weight_passes = (int64_t)s[1];
  m->stats.candidates = (int64_t)s[2];
  m->stats.beam_steps = (int64_t)s[3];
  m->stats.max_k = (int32_t)s[4];
  if (int rc = event_times(m)) return rc;
  m->stats_pending = false;
  std::vector<int> status(m->last_U);
  CU(cudaMemcpy(status.data(), m->status.p, (size_t)m->last_U * sizeof(int), cudaMemcpyDeviceToHost));
  int overflow = 0, bad = 0, capacity = 0;
  for (int v : status) {
    if (v == -4) ++overflow;
    else if (v == -5) ++capacity;
    else if (v != 0) ++bad;
  }
  if (capacity && m->last_tree_spill)
    return fail(UIS_ERR_CAPACITY, "%d utterance(s): the look-ahead tree of one beam step exhausted the device-memory arena "
                "(%d nodes / %d leaves per CTA from a budget of %zu MiB; raise UISRNN_B200_TREE_SPILL_MB or lower "
                "beam_size / look_ahead / kcap)", capacity, m->last_spill_ni, m->last_spill_nlf, m->last_spill_budget >> 20);
  if (capacity)
    return fail(UIS_ERR_CAPACITY, "%d utterance(s): the look-ahead tree of one beam step outgrew the on-chip node arrays "
                "(lower beam_size / look_ahead / kcap)", capacity);
  if (overflow)
    return fail(UIS_ERR_OVERFLOW, "%d utterance(s) opened more clusters than kcap; retry with a larger kcap", overflow);
  if (bad) return fail(UIS_ERR_INVALID, "%d utterance(s) ended with no finite hypothesis", bad);
  return 0;
}

// Zero-pads the caller's `rows` device rows (D_user wide) to the kernel's row length D in m->x32 and points *x_dev
// there; a model whose D_user is the kernel's D is left alone.
int pad_to_kernel_d(uis_model* m, const float** x_dev, size_t rows, cudaStream_t st) {
  if (m->D == m->D_user || rows == 0) return 0;
  if (int rc = m->x32.ensure(rows * m->D * 4)) return rc;
  const size_t np = rows * m->D;
  const int blocks = (int)std::min<size_t>((np + 255) / 256, (size_t)m->num_sms * 16);
  uis::pad_rows_f32_kernel<<<blocks, 256, 0, st>>>(*x_dev, m->x32.as<float>(), rows, m->D_user, m->D);
  CU(cudaGetLastError());
  *x_dev = m->x32.as<float>();
  return 0;
}

// A failed call may leave copies / kernels in flight on either stream: drain them (the error already recorded in
// uis_last_error() is the one reported) so that the staging ring and the workspace are quiescent for the next call.
void drain_after_failure(uis_model* m, cudaStream_t st) {
  const std::string keep = g_err;
  if (m->copy_stream) cudaStreamSynchronize(m->copy_stream);
  cudaStreamSynchronize(st);
  (void)cudaGetLastError();
  g_err = keep;
}

// Orders one call's device work after the previous call's on the same handle.  Every call shares the handle's
// workspace (gi, slot pools, chain plans, ...), so a call on another stream could overwrite it while the previous
// call's kernels still read it.  Constructed before the call's first enqueue: `st` waits for the event the previous
// call recorded at its end (cudaStreamWaitEvent: the host does not block; on the previous call's own stream the wait
// adds nothing).  Destroyed when the call returns: records that event on `st`.
class CallOrder {
 public:
  CallOrder(uis_model* m, cudaStream_t st) : m_(m), st_(st) {
    if (!m->ev_done) status = cudaEventCreateWithFlags(&m->ev_done, cudaEventDisableTiming);
    else if (m->done_recorded) status = cudaStreamWaitEvent(st, m->ev_done, 0);
  }
  ~CallOrder() {
    if (m_->ev_done) m_->done_recorded = cudaEventRecord(m_->ev_done, st_) == cudaSuccess;
  }
  cudaError_t status = cudaSuccess;

 private:
  uis_model* m_;
  cudaStream_t st_;
};

// A device-buffer decode in the groups `cuts` (cut_groups), one after the other on `st`, nothing read back.  Group
// [u0, u1) reads its rows from x_dev + off[u0] rows, padded to the kernel's D in the handle's x32 when the model is
// padded, so that its float4 loads start on a 16-byte boundary either way (an unpadded row is a multiple of 64
// floats).  Its label planes start at row off[u0] of the call's [C][k][rows] planes (rows = plane apart); its
// per-job outputs land in the handle's buffers and one 2-D copy per output puts their [C][u1 - u0] blocks at column
// u0 of the caller's [C][U][k] / [C][U] arrays.  Its jobs' status sits at [u0 * C, u1 * C) of the handle's, which
// collect() reads for the whole call.
int predict_device_groups(uis_model* m, const float* x_dev, const int64_t* off, int U, long long plane,
                          const uis_predict_opts* opts, int32_t* labels_dev, cudaStream_t st, const SpeakerBounds& sb,
                          const NBestOut& nb, const DecodeParams& dp, const std::vector<int>& cuts) {
  const int C = dp.count, K = nb.k, G = (int)cuts.size() - 1;
  size_t max_jobs = 0;
  for (int g = 0; g < G; ++g) max_jobs = std::max(max_jobs, (size_t)(cuts[g + 1] - cuts[g]) * C);
  NBestOut gnb{K};
  if (nb.scores) {
    if (int rc = m->nb_scores.ensure(max_jobs * K * 4)) return rc;
    gnb.scores = m->nb_scores.as<float>();
  }
  if (nb.speakers) {
    if (int rc = m->nb_speakers.ensure(max_jobs * K * 4)) return rc;
    gnb.speakers = m->nb_speakers.as<int32_t>();
  }
  if (nb.count) {
    if (int rc = m->nb_count.ensure(max_jobs * 4)) return rc;
    gnb.count = m->nb_count.as<int32_t>();
  }
  if (int rc = m->status.ensure((size_t)U * C * sizeof(int))) return rc;
  CU(cudaMemsetAsync(m->status.p, 0, (size_t)U * C * sizeof(int), st));  // a group of empty utterances launches nothing
  uis_stats total{};
  int ran = 0;
  for (int g = 0; g < G; ++g) {
    const int u0 = cuts[g], u1 = cuts[g + 1], Ug = u1 - u0;
    const std::vector<int64_t> goff = group_offsets(off, u0, u1);
    Plan gp;
    if (int rc = make_plan(m, goff.data(), Ug, opts, &gp, C)) return rc;
    const float* gx = x_dev + (size_t)off[u0] * m->D_user;
    if (int rc = pad_to_kernel_d(m, &gx, (size_t)gp.rows, st)) return rc;
    if (int rc = run_device(m, gx, goff.data(), Ug, gp, labels_dev + off[u0], nullptr, st, sb.at(u0), gnb, dp, false,
                            Group{ran, u0 * C, plane, 0}))
      return rc;
    ran += gp.rows > 0 ? 1 : 0;
    const size_t w = (size_t)Ug * K * 4;  // one config's block of the group: [Ug][k]
    if (nb.scores)
      CU(cudaMemcpy2DAsync(nb.scores + (size_t)u0 * K, (size_t)U * K * 4, gnb.scores, w, w, C, cudaMemcpyDeviceToDevice, st));
    if (nb.speakers)
      CU(cudaMemcpy2DAsync(nb.speakers + (size_t)u0 * K, (size_t)U * K * 4, gnb.speakers, w, w, C,
                           cudaMemcpyDeviceToDevice, st));
    if (nb.count)
      CU(cudaMemcpy2DAsync(nb.count + u0, (size_t)U * 4, gnb.count, (size_t)Ug * 4, (size_t)Ug * 4, C,
                           cudaMemcpyDeviceToDevice, st));
    add_stats(&total, m->stats);
  }
  m->stats = total;
  m->last_U = U * C;
  m->last_groups = ran;
  m->stats_pending = ran > 0;
  return 0;
}

int predict_device_impl(uis_model* m, const float* x_dev, const int64_t* frame_offsets, int U,
                        const uis_predict_opts* opts, int32_t* labels_dev, const uis_debug_taps* taps, void* stream,
                        const int32_t* max_speakers, const int32_t* min_speakers, int32_t* speakers_dev,
                        const NBestOut& nb, const DecodeParams* dpp = nullptr) {
  if (!m) return fail(UIS_ERR_INVALID, "model is NULL");
  const DecodeParams dp = dpp ? *dpp : model_decode(m);
  Plan pl;
  if (int rc = make_plan(m, frame_offsets, U, opts, &pl, dp.count)) return rc;
  if (int rc = check_bounds(U, max_speakers, min_speakers)) return rc;
  if (U > 0 && pl.rows > 0 && (!x_dev || !labels_dev)) return fail(UIS_ERR_INVALID, "null device buffer");
  uis::DeviceGuard device_guard_(m->device);
  CU(device_guard_.status);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  CallOrder order(m, st);
  CU(order.status);
  // Memory: the rows and the label planes are the caller's; per frame the call holds gi (12H B) and, for a model
  // padded to its kernel shape, the padded fp32 rows (4D B).
  const bool padded = m->D != m->D_user;
  const size_t per_row = (size_t)3 * m->H * 4 + (padded ? (size_t)m->D * 4 : 0);
  const size_t fixed = workspace_bytes(m, pl, U, dp.count) - (size_t)pl.rows * 3 * m->H * 4;
  size_t max_rows = 0;
  if (int rc = row_budget(per_row, fixed, m->gi.cap + (padded ? m->x32.cap : 0), &max_rows)) return rc;
  const SpeakerBounds sb{max_speakers, min_speakers, speakers_dev};
  if ((size_t)pl.rows > max_rows && !taps && U > 1)
    return predict_device_groups(m, x_dev, frame_offsets, U, pl.rows, opts, labels_dev, st, sb, nb, dp,
                                 cut_groups(frame_offsets, U, max_rows));
  if (int rc = pad_to_kernel_d(m, &x_dev, (size_t)pl.rows, st)) return rc;
  return run_device(m, x_dev, frame_offsets, U, pl, labels_dev, taps, st, sb, nb, dp);
}

// ---- host input pipeline -----------------------------------------------------------------------------------------

int ensure_host_path(uis_model* m) {
  if (!m->copy_stream) CU(cudaStreamCreateWithFlags(&m->copy_stream, cudaStreamNonBlocking));
  for (int i = 0; i < uis_model::kSlots; ++i) {
    if (!m->ev_copied[i]) CU(cudaEventCreateWithFlags(&m->ev_copied[i], cudaEventDisableTiming));
    if (!m->ev_free[i]) CU(cudaEventCreateWithFlags(&m->ev_free[i], cudaEventDisableTiming));
  }
  for (auto& e : m->ev_h2d)
    if (!e) CU(cudaEventCreate(&e));
  if (!m->ev_pipe) CU(cudaEventCreate(&m->ev_pipe));
  for (auto& e : m->ev)
    if (!e) CU(cudaEventCreate(&e));
  return 0;
}

// Rows of one staging chunk of the host-buffer path (UISRNN_B200_CHUNK_MB of float64, default 32 MB: long enough
// for full PCIe rate, short enough that the first cast starts ~0.6 ms after the call).
size_t staging_chunk_rows(int d_user) {
  long long mb = 32;
  if (const char* env = std::getenv("UISRNN_B200_CHUNK_MB")) mb = std::max(0ll, std::atoll(env));  // 0 = the 256-row floor
  return std::max<size_t>(256, (size_t)mb * (1u << 20) / ((size_t)d_user * 8));
}

// Input pipeline of the host-buffer entry points (uis_predict*, uis_score): the float64 rows of utterances [0, U)
// (device rows off[u] ..) travel in chunks through the staging ring on the copy stream while `st` casts each landed
// chunk to fp32 (padded to m->D) into m->x32 and runs its input projection into m->gi.  ev_h2d[0..1] bracket the
// copies, ev_pipe marks the first cast.
int stage_host_rows(uis_model* m, const double* const* seqs, int U, const int64_t* off, size_t rows, cudaStream_t st,
                    int* n_chunks_out, bool* staged_out) {
  const int D = m->D_user, H = m->H;
  if (int rc = ensure_host_path(m)) return rc;
  const size_t chunk = std::min(staging_chunk_rows(D), rows);
  const int n_chunks = (int)((rows + chunk - 1) / chunk);
  const int slots = std::min(n_chunks, (int)uis_model::kSlots);
  if (int rc = m->x64.ensure((size_t)slots * chunk * D * 8)) return rc;
  if (int rc = m->x32.ensure(rows * m->D * 4)) return rc;
  if (int rc = m->gi.ensure(rows * 3 * H * sizeof(float))) return rc;
  cudaStream_t cs = m->copy_stream;
  // Pageable or pinned?  Ordinary numpy arrays are pageable: the driver would stage every cudaMemcpy itself, in one
  // thread (measured 10.8 GB/s against 44.6 GB/s from pinned memory).  Such inputs go through a pinned ring of our own,
  // filled by a few host threads while the previous chunk is on the bus.  UISRNN_B200_HOST_STAGING=0 / 1 overrides.
  bool staged = false;
  {
    const char* env = std::getenv("UISRNN_B200_HOST_STAGING");
    if (env && (env[0] == '0' || env[0] == '1')) {
      staged = env[0] == '1';
    } else if (rows * (size_t)D * 8 >= ((size_t)8 << 20)) {  // small inputs: not worth waking the threads
      for (int q = 0; q < U && !staged; q += std::max(1, U / 8)) {  // a sample of the list
        if (off[q + 1] <= off[q]) continue;
        cudaPointerAttributes attr{};
        if (cudaPointerGetAttributes(&attr, seqs[q]) != cudaSuccess) { (void)cudaGetLastError(); staged = true; }
        else if (attr.type == cudaMemoryTypeUnregistered) staged = true;
      }
    }
  }
  const size_t chunk_bytes = chunk * (size_t)D * 8;
  if (staged) {
    if ((size_t)slots * chunk_bytes > m->pin_stage_cap) {
      if (m->pin_stage) cudaFreeHost(m->pin_stage);
      m->pin_stage = nullptr;
      m->pin_stage_cap = 0;
      if (cudaMallocHost(&m->pin_stage, (size_t)slots * chunk_bytes) != cudaSuccess) {
        (void)cudaGetLastError();
        staged = false;  // no pinned memory to be had: let the driver stage the copies
      } else {
        m->pin_stage_cap = (size_t)slots * chunk_bytes;
      }
    }
    for (auto& e : m->ev_dma)
      if (!e) CU(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    if (staged && !m->copy_pool) {
      const unsigned hw = std::max(1u, std::thread::hardware_concurrency());
      int nthreads = (int)std::min(16u, std::max(2u, hw / 2));  // more threads fill the staging ring faster
      if (const char* env = std::getenv("UISRNN_B200_COPY_THREADS")) nthreads = std::max(1, std::min(64, std::atoi(env)));
      m->copy_pool = new CopyPool(nthreads);
    }
  }
  CU(cudaEventRecord(m->ev_h2d[0], cs));
  CU(cudaEventRecord(m->ev_pipe, st));
  size_t r0 = 0;
  int u = 0;
  std::vector<CopyPiece> pieces;
  for (int c = 0; r0 < rows; ++c) {
    const size_t r1 = std::min(rows, r0 + chunk);
    const int slot = c % uis_model::kSlots;
    double* stage = m->x64.as<double>() + (size_t)slot * chunk * D;
    if (staged) {
      pieces.clear();
      for (size_t r = r0; r < r1;) {
        while (u < U && (size_t)off[u + 1] <= r) ++u;
        const size_t take = std::min((size_t)off[u + 1], r1) - r;
        pieces.push_back(CopyPiece{reinterpret_cast<const char*>(seqs[u] + (r - (size_t)off[u]) * D), (r - r0) * D * 8, take * D * 8});
        r += take;
      }
      char* pin = m->pin_stage + (size_t)slot * chunk_bytes;
      if (c >= uis_model::kSlots) CU(cudaEventSynchronize(m->ev_dma[slot]));  // the DMA out of this pinned slot is done
      m->copy_pool->run(&pieces, pin, (r1 - r0) * D * 8);
      if (c >= uis_model::kSlots) CU(cudaStreamWaitEvent(cs, m->ev_free[slot], 0));
      CU(cudaMemcpyAsync(stage, pin, (r1 - r0) * D * 8, cudaMemcpyHostToDevice, cs));
      CU(cudaEventRecord(m->ev_dma[slot], cs));
    } else {
      if (c >= uis_model::kSlots) CU(cudaStreamWaitEvent(cs, m->ev_free[slot], 0));  // cast of chunk c - kSlots has read the slot
      for (size_t r = r0; r < r1;) {
        while (u < U && (size_t)off[u + 1] <= r) ++u;  // the utterance that holds row r (empty ones are skipped)
        const size_t take = std::min((size_t)off[u + 1], r1) - r;
        CU(cudaMemcpyAsync(stage + (r - r0) * D, seqs[u] + (r - (size_t)off[u]) * D, take * D * 8, cudaMemcpyHostToDevice, cs));
        r += take;
      }
    }
    CU(cudaEventRecord(m->ev_copied[slot], cs));
    CU(cudaStreamWaitEvent(st, m->ev_copied[slot], 0));
    const size_t nr = r1 - r0, np = nr * m->D;
    const int blocks = (int)std::min<size_t>((np + 255) / 256, (size_t)m->num_sms * 16);
    float* x32 = m->x32.as<float>() + r0 * m->D;
    if (m->D == D) uis::cast_f64_f32_kernel<<<blocks, 256, 0, st>>>(stage, x32, np);
    else uis::cast_pad_f64_f32_kernel<<<blocks, 256, 0, st>>>(stage, x32, nr, D, m->D);
    dim3 grid((3 * H + uis::PBN - 1) / uis::PBN, (unsigned)((nr + uis::PBM - 1) / uis::PBM));
    uis::input_proj_kernel<<<grid, 256, 0, st>>>(x32, m->wih_t.as<float>(), m->bih.as<float>(),
                                                m->gi.as<float>() + r0 * 3 * H, (int)nr, 3 * H, m->D);
    CU(cudaGetLastError());
    CU(cudaEventRecord(m->ev_free[slot], st));
    r0 = r1;
  }
  CU(cudaEventRecord(m->ev_h2d[1], cs));
  *n_chunks_out = n_chunks;
  *staged_out = staged;
  return 0;
}

// One group of utterances, host buffers in, host buffers out: chunked H2D on the copy stream || cast + input
// projection on `st`, then the beam kernel, then one D2H copy of all labels.
int predict_host_group_impl(uis_model* m, const double* const* seqs, const int64_t* n_frames, int U, const int64_t* off,
                            const Plan& pl, int32_t* const* labels_out, const uis_debug_taps* taps, cudaStream_t st,
                            const SpeakerBounds& sb_host, int32_t* speakers_out, const NBestOut& nb_host, int u0,
                            int U_all, const DecodeParams& dp) {
  const size_t rows = (size_t)pl.rows;
  const int C = dp.count, J = U * C;
  if (rows == 0) {
    m->stats = uis_stats{};
    m->stats.utterances = J;
    return 0;
  }
  const int K = nb_host.k;
  const size_t planes = (size_t)K * C;  // label planes: [config][hypothesis]
  if (int rc = m->labels.ensure(rows * 4 * planes)) return rc;
  SpeakerBounds sb = sb_host;  // speaker counts land in the handle's device buffer, then in `speakers_out`
  if (speakers_out) {
    if (int rc = m->spk_out.ensure((size_t)U * 4)) return rc;
    sb.out_dev = m->spk_out.as<int32_t>();
  }
  NBestOut nb{K};  // likewise the N-best scores, cluster counts and hypothesis counts
  if (nb_host.scores) {
    if (int rc = m->nb_scores.ensure((size_t)J * K * 4)) return rc;
    nb.scores = m->nb_scores.as<float>();
  }
  if (nb_host.speakers) {
    if (int rc = m->nb_speakers.ensure((size_t)J * K * 4)) return rc;
    nb.speakers = m->nb_speakers.as<int32_t>();
  }
  if (nb_host.count) {
    if (int rc = m->nb_count.ensure((size_t)J * 4)) return rc;
    nb.count = m->nb_count.as<int32_t>();
  }
  if (rows * 4 * planes > m->labels_pin_cap) {
    if (m->labels_pin) cudaFreeHost(m->labels_pin);
    m->labels_pin = nullptr;
    m->labels_pin_cap = 0;
    const size_t want = rows * 4 * planes + rows / 2 + 4096;
    if (cudaMallocHost(&m->labels_pin, want) != cudaSuccess) {
      (void)cudaGetLastError();
      return fail(UIS_ERR_NOMEM, "cudaMallocHost(%zu) for the label staging buffer failed", want);
    }
    m->labels_pin_cap = want;
  }
  int n_chunks = 0;
  bool staged = false;
  if (int rc = stage_host_rows(m, seqs, U, off, rows, st, &n_chunks, &staged)) return rc;
  if (int rc = run_device(m, m->x32.as<float>(), off, U, pl, m->labels.as<int32_t>(), taps, st, sb, nb, dp,
                         /*gi_ready=*/true))
    return rc;
  m->stats.kernel_launches = 1 + 2 * (int64_t)n_chunks + (pl.kernel == uis::Kernel::Tree && pl.spill_ctas ? 1 : 0);
  m->stats.chunks = n_chunks;
  m->stats.staged = staged ? 1 : 0;
  CU(cudaMemcpyAsync(m->labels_pin, m->labels.p, rows * 4 * planes, cudaMemcpyDeviceToHost, st));
  CU(cudaStreamSynchronize(st));
  for (size_t j = 0; j < planes; ++j)  // plane j of the device rows -> rows j of the caller's [C][K][n_frames[q]] buffers
    for (int q = 0; q < U; ++q)
      if (n_frames[q] > 0)
        std::memcpy(labels_out[q] + j * n_frames[q], m->labels_pin + j * rows + off[q], (size_t)n_frames[q] * 4);
  if (speakers_out) CU(cudaMemcpy(speakers_out, sb.out_dev, (size_t)U * 4, cudaMemcpyDeviceToHost));
  for (int c = 0; c < C; ++c) {  // config c's block of this group -> [c][u0 ..][K] of the whole list's outputs
    const size_t dst = (size_t)c * U_all + u0, src = (size_t)c * U;
    if (nb.scores) CU(cudaMemcpy(nb_host.scores + dst * K, nb.scores + src * K, (size_t)U * K * 4, cudaMemcpyDeviceToHost));
    if (nb.speakers)
      CU(cudaMemcpy(nb_host.speakers + dst * K, nb.speakers + src * K, (size_t)U * K * 4, cudaMemcpyDeviceToHost));
    if (nb.count) CU(cudaMemcpy(nb_host.count + dst, nb.count + src, (size_t)U * 4, cudaMemcpyDeviceToHost));
  }
  if (int rc = collect(m)) return rc;
  CU(cudaEventElapsedTime(&m->stats.h2d_ms, m->ev_h2d[0], m->ev_h2d[1]));
  CU(cudaEventElapsedTime(&m->stats.pipeline_ms, m->ev_pipe, m->ev[1]));  // first cast -> beam kernel start
  return 0;
}

// Utterances [u0, u0 + U) of a list of U_all; `nb` holds the whole list's [configs][U_all][k] outputs.
int predict_host_group(uis_model* m, const double* const* seqs, const int64_t* n_frames, int U, const int64_t* off,
                       const Plan& pl, int32_t* const* labels_out, const uis_debug_taps* taps, cudaStream_t st,
                       const SpeakerBounds& sb, int32_t* speakers_out, const NBestOut& nb, int u0, int U_all,
                       const DecodeParams& dp) {
  const int rc = predict_host_group_impl(m, seqs, n_frames, U, off, pl, labels_out, taps, st, sb, speakers_out, nb, u0,
                                         U_all, dp);
  if (rc != 0 && rc != UIS_ERR_OVERFLOW && rc != UIS_ERR_CAPACITY) drain_after_failure(m, st);
  return rc;
}

int predict_host_impl(uis_model* m, const double* const* seqs, const int64_t* n_frames, int U,
                      const uis_predict_opts* opts, int32_t* const* labels_out, const uis_debug_taps* taps, void* stream,
                      const int32_t* max_speakers, const int32_t* min_speakers, int32_t* speakers_out,
                      const NBestOut& nb, const DecodeParams* dpp = nullptr) {
  if (!m) return fail(UIS_ERR_INVALID, "model is NULL");
  if (U < 0 || (U > 0 && (!seqs || !n_frames || !labels_out))) return fail(UIS_ERR_INVALID, "null argument");
  if (int rc = check_bounds(U, max_speakers, min_speakers)) return rc;
  const DecodeParams dp = dpp ? *dpp : model_decode(m);
  const size_t J = (size_t)U * dp.count;
  if (speakers_out && U > 0) std::memset(speakers_out, 0, (size_t)U * sizeof(int32_t));  // empty inputs: 0
  if (U > 0) {  // empty inputs return no N-best hypothesis
    if (nb.scores) std::fill(nb.scores, nb.scores + J * nb.k, std::numeric_limits<float>::infinity());
    if (nb.speakers) std::memset(nb.speakers, 0, J * nb.k * sizeof(int32_t));
    if (nb.count) std::memset(nb.count, 0, J * sizeof(int32_t));
  }
  const auto t_begin = std::chrono::steady_clock::now();
  std::vector<int64_t> off(U + 1, 0);
  for (int u = 0; u < U; ++u) {
    if (n_frames[u] < 0) return fail(UIS_ERR_INVALID, "negative length");
    if (n_frames[u] > 0 && (!seqs[u] || !labels_out[u])) return fail(UIS_ERR_INVALID, "null utterance buffer");
    off[u + 1] = off[u] + n_frames[u];
  }
  Plan pl;
  if (int rc = make_plan(m, off.data(), U, opts, &pl, dp.count)) return rc;
  uis::DeviceGuard device_guard_(m->device);
  CU(device_guard_.status);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (pl.rows == 0) return 0;
  CallOrder order(m, st);
  CU(order.status);
  // Memory: the per-frame workspace (gi 12H B + fp32 rows 4D B + labels) is the part that grows with the input.
  // A list that does not fit the device at once is decoded in groups of whole utterances (row_budget, cut_groups).
  const size_t per_row = (size_t)3 * m->H * 4 + (size_t)m->D * 4 + (size_t)4 * nb.k * dp.count;  // (+ one label per plane)
  const size_t held = m->gi.cap + m->x32.cap + m->labels.cap + m->x64.cap;  // re-used by this call
  const size_t fixed = workspace_bytes(m, pl, U, dp.count) - (size_t)pl.rows * 3 * m->H * 4 +
                       (size_t)uis_model::kSlots * staging_chunk_rows(m->D_user) * m->D_user * 8 + J * (2 * nb.k + 1) * 4;
  size_t max_rows = 0;
  if (int rc = row_budget(per_row, fixed, held, &max_rows)) return rc;
  if ((size_t)pl.rows <= max_rows || taps || U <= 1) {
    if (int rc = predict_host_group(m, seqs, n_frames, U, off.data(), pl, labels_out, taps, st,
                                    SpeakerBounds{max_speakers, min_speakers}, speakers_out, nb, 0, U, dp))
      return rc;
    m->stats.groups = 1;
  } else {
    uis_stats total{};
    const std::vector<int> cuts = cut_groups(off.data(), U, max_rows);
    for (size_t g = 0; g + 1 < cuts.size(); ++g) {
      const int u0 = cuts[g], u1 = cuts[g + 1];
      const std::vector<int64_t> goff = group_offsets(off.data(), u0, u1);
      Plan gp;
      if (int rc = make_plan(m, goff.data(), u1 - u0, opts, &gp, dp.count)) return rc;
      if (int rc = predict_host_group(m, seqs + u0, n_frames + u0, u1 - u0, goff.data(), gp, labels_out + u0, nullptr, st,
                                      SpeakerBounds{max_speakers, min_speakers}.at(u0),
                                      speakers_out ? speakers_out + u0 : nullptr, nb, u0, U, dp))
        return rc;
      m->stats.groups = 1;
      add_stats(&total, m->stats);
    }
    m->stats = total;
  }
  m->stats.host_ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t_begin).count();
  return 0;
}

// ---- score(): the neg_likelihood of given labellings (uis_kernels_score.cu) ----------------------------------------

// Chains of a score call, one per (utterance, cluster), longest first, with their frame rows in frame order.  The
// labels must be canonical: 0, 1, 2, ... in order of first appearance (the ids a trace holds).
struct ChainPlan {
  std::vector<long long> off, rows;  // [chains + 1] offsets into rows; [frames] device rows
  int chains = 0, queued = 0, max_k = 0;  // queued: chains of length >= 2 (a prefix, longest first)
};

int plan_chains(const int32_t* labels, const int64_t* off, int U, ChainPlan* cp, int u_base = 0) {
  std::vector<long long> base(U + 1, 0);  // first chain id of every utterance
  for (int u = 0; u < U; ++u) {
    int K = 0;
    for (long long r = off[u]; r < off[u + 1]; ++r) {
      const int c = labels[r];
      if (c < 0 || c > K)
        return fail(UIS_ERR_INVALID, "utterance %d frame %lld: label %d is not canonical (labels are 0, 1, 2, ... in "
                    "order of first appearance, so at most %d here)", u_base + u, r - off[u], c, K);
      K += (c == K) ? 1 : 0;
    }
    base[u + 1] = base[u] + K;
    cp->max_k = std::max(cp->max_k, K);
  }
  const long long nch = base[U], rows = U > 0 ? off[U] : 0;
  if (nch > 0x7fffffffll) return fail(UIS_ERR_INVALID, "more than 2^31 - 1 (utterance, cluster) chains");
  std::vector<long long> len(nch, 0);
  for (int u = 0; u < U; ++u)
    for (long long r = off[u]; r < off[u + 1]; ++r) ++len[base[u] + labels[r]];
  std::vector<int> order(nch);
  std::iota(order.begin(), order.end(), 0);
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return len[a] > len[b]; });
  cp->off.assign(nch + 1, 0);
  std::vector<long long> cursor(nch);
  for (long long i = 0; i < nch; ++i) {
    cp->off[i + 1] = cp->off[i] + len[order[i]];
    cursor[order[i]] = cp->off[i];
  }
  cp->rows.resize(std::max(rows, 1ll));
  for (int u = 0; u < U; ++u)
    for (long long r = off[u]; r < off[u + 1]; ++r) cp->rows[cursor[base[u] + labels[r]]++] = r;
  cp->chains = (int)nch;
  cp->queued = 0;
  while (cp->queued < cp->chains && len[order[cp->queued]] >= 2) ++cp->queued;
  return 0;
}

// Enqueues a score call on `st`: input projection (unless gi_ready), chain kernel, first visits, then one reduce per
// config of `dp` (scores_dev [configs][U], frame_dev [configs][rows]; a group of a larger call: rows grp.stride and
// grp.plane apart).  x_dev: the fp32 rows at the kernel shape (m->D); labels_dev: the canonical labels the plan was
// made from.  cp: a host plan, uploaded here; nullptr: the device plan that score_plan wrote to sc_chain_off /
// sc_chain_rows / the group's sc_counts earlier on `st` (row_off is on the device too).
int run_score(uis_model* m, const float* x_dev, const int64_t* off, int U, const ChainPlan* cp, const int32_t* labels_dev,
              float* scores_dev, float* frame_dev, cudaStream_t st, bool gi_ready, const DecodeParams& dp,
              const Group& grp = Group{}) {
  const int H = m->H, D = m->D;
  const long long rows = off[U];
  long long maxN = 0;
  for (int u = 0; u < U; ++u) maxN = std::max<long long>(maxN, off[u + 1] - off[u]);
  uis::ScoreParams sp{};
  sp.b = model_params(m);
  if (int rc = ensure_log_tables(m, (int)maxN, dp, &sp.b)) return rc;  // block counts and totals reach N
  if (uis::score_smem(H, D) > uis::kSmemCap) return fail(UIS_ERR_UNSUPPORTED, "no score kernel for hidden=%d dim=%d", H, D);
  int CP = 0;  // columns per pass: the FFMA beam kernel's
  uis::with_shape(uis::AllShapes{}, H, D, [&](auto s) { CP = uis::beam_cp<decltype(s)::H>(); });
  // a device plan's counts are not known here: the grids are sized from their bounds (every queued chain has two frames)
  const long long queued = cp ? cp->queued : rows / 2;
  const int ctas = (int)std::max(1ll, std::min<long long>(m->num_sms, (queued + CP - 1) / CP));
  if (int rc = m->row_off.ensure((U + 1) * sizeof(long long))) return rc;
  if (int rc = m->queue_stats.ensure(40 * sizeof(unsigned long long))) return rc;
  if (int rc = m->gi.ensure((size_t)rows * 3 * H * sizeof(float))) return rc;
  if (int rc = m->pool_mean.ensure((size_t)ctas * CP * 2 * D * sizeof(float))) return rc;
  if (int rc = m->pool_hidden.ensure((size_t)ctas * CP * 2 * m->depth * H * sizeof(float))) return rc;
  if (int rc = m->sc_mse.ensure((size_t)rows * sizeof(float))) return rc;
  if (int rc = m->sc_blocks.ensure((size_t)rows * sizeof(int))) return rc;
  if (cp) {
    if (int rc = m->sc_chain_off.ensure(cp->off.size() * sizeof(long long))) return rc;
    if (int rc = m->sc_chain_rows.ensure(cp->rows.size() * sizeof(long long))) return rc;
    std::vector<long long> off_ll(off, off + U + 1);
    CU(cudaMemcpyAsync(m->row_off.p, off_ll.data(), (U + 1) * sizeof(long long), cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(m->sc_chain_off.p, cp->off.data(), cp->off.size() * sizeof(long long), cudaMemcpyHostToDevice, st));
    CU(cudaMemcpyAsync(m->sc_chain_rows.p, cp->rows.data(), cp->rows.size() * sizeof(long long), cudaMemcpyHostToDevice,
                       st));
  }
  CU(cudaMemsetAsync(m->queue_stats.p, 0, grp.index ? kQueueBytes : 40 * sizeof(unsigned long long), st));

  sp.b.x = x_dev; sp.b.gi = m->gi.as<float>();
  sp.b.row_off = m->row_off.as<long long>();
  sp.b.U = U; sp.b.n_utt = U; sp.b.P = 2;
  sp.b.pool_mean = m->pool_mean.as<float>(); sp.b.pool_hidden = m->pool_hidden.as<float>();
  sp.b.queue = m->queue_stats.as<int>();
  sp.b.stats = m->queue_stats.as<unsigned long long>() + 8;
  sp.chain_off = m->sc_chain_off.as<long long>(); sp.chain_rows = m->sc_chain_rows.as<long long>();
  sp.chains = cp ? cp->chains : (int)rows; sp.queued = (int)queued;
  sp.counts = cp ? nullptr : m->sc_counts.as<int>() + 4 * grp.index;
  sp.mse = m->sc_mse.as<float>(); sp.labels = labels_dev; sp.scores = scores_dev; sp.frame_out = frame_dev;
  sp.score_stride = grp.stride ? grp.stride : U;
  sp.frame_stride = grp.plane ? grp.plane : rows;
  sp.blocks = m->sc_blocks.as<int>();

  if (int rc = group_events(m, grp.index)) return rc;
  cudaEvent_t* ev = m->ev.data() + 3 * grp.index;
  CU(cudaEventRecord(ev[0], st));
  if (!gi_ready) {
    dim3 grid((3 * H + uis::PBN - 1) / uis::PBN, (unsigned)((rows + uis::PBM - 1) / uis::PBM));
    uis::input_proj_kernel<<<grid, 256, 0, st>>>(x_dev, m->wih_t.as<float>(), m->bih.as<float>(), m->gi.as<float>(),
                                                (int)rows, 3 * H, D);
    CU(cudaGetLastError());
  }
  CU(cudaEventRecord(ev[1], st));
  cudaError_t e = cudaSuccess;
  if (queued > 0) {
    if (!uis::launch_score_chains(H, D, sp, ctas, st, &e))
      return fail(UIS_ERR_UNSUPPORTED, "no score kernel for hidden=%d dim=%d", H, D);
    if (e != cudaSuccess) return fail(UIS_ERR_CUDA, "score chain kernel launch failed: %s", cudaGetErrorString(e));
  }
  CU(cudaEventRecord(ev[2], st));
  if (!uis::launch_score_first(H, D, sp, st, &e)) return fail(UIS_ERR_UNSUPPORTED, "no score kernel for dim=%d", D);
  if (e != cudaSuccess) return fail(UIS_ERR_CUDA, "score first-visit kernel launch failed: %s", cudaGetErrorString(e));
  for (int c = 0; c < dp.count; ++c) {  // the Gaussian terms in sc_mse serve every config
    e = uis::launch_score_reduce(sp, c, st);
    if (e != cudaSuccess) return fail(UIS_ERR_CUDA, "score reduce kernel launch failed: %s", cudaGetErrorString(e));
  }
  m->stats.ctas = queued > 0 ? ctas : 0;
  m->stats.kernel_launches = (gi_ready ? 0 : 1) + (queued > 0 ? 1 : 0) + 1 + dp.count;
  m->stats_pending = true;
  return 0;
}

// Stats of a score call before it runs (the rest is zero; collect() adds the chain kernel's counters and times).
void begin_score_stats(uis_model* m, int jobs, long long rows, const ChainPlan& cp, cudaStream_t st) {
  m->stats = uis_stats{};
  m->stats.utterances = jobs;
  m->stats.frames = rows;
  m->stats.max_k = cp.max_k;
  m->stats.engine = 1;
  m->stats.groups = 1;
  m->last_U = jobs;
  m->last_groups = 1;
  m->last_score = true;
  m->last_score_counts = false;
  m->last_tree_spill = false;
  m->last_stream = st;
  m->stats_pending = false;
}

// Per-frame bytes of a score call's device workspace: gi (12H), the Gaussian term and block count of every frame,
// the chain plan (an offset and a row), and the fp32 rows at the kernel shape when the call holds them (staged host
// rows, or a padded model's device rows).  *held: what the handle's buffers of those already hold.
size_t score_row_bytes(const uis_model* m, bool x32, size_t* held) {
  *held = m->gi.cap + m->sc_mse.cap + m->sc_blocks.cap + m->sc_chain_off.cap + m->sc_chain_rows.cap + (x32 ? m->x32.cap : 0);
  return (size_t)3 * m->H * 4 + 4 + 4 + 8 + 8 + (x32 ? (size_t)m->D * 4 : 0);
}

// Bytes of a score call over U utterances and C configs that do not grow with the frames: the chain kernel's slot
// pools at its largest grid, the offsets and the totals.
size_t score_fixed_bytes(const uis_model* m, int U, int C) {
  int CP = 0;
  uis::with_shape(uis::AllShapes{}, m->H, m->D, [&](auto s) { CP = uis::beam_cp<decltype(s)::H>(); });
  return (size_t)m->num_sms * CP * 2 * (m->D + (size_t)m->depth * m->H) * 4 + (size_t)(U + 1) * 8 + (size_t)U * C * 4;
}

// Chain plans of the groups `cuts` of a host-planned score call (offsets `off`, canonical labels `lab` of every row),
// each over its group's own rows.  Made before any group runs, so that a bad label fails the call before it enqueues.
int plan_groups(const int32_t* lab, const int64_t* off, const std::vector<int>& cuts, std::vector<ChainPlan>* plans) {
  plans->resize(cuts.size() - 1);
  for (size_t g = 0; g + 1 < cuts.size(); ++g) {
    const std::vector<int64_t> goff = group_offsets(off, cuts[g], cuts[g + 1]);
    if (int rc = plan_chains(lab + off[cuts[g]], goff.data(), cuts[g + 1] - cuts[g], &(*plans)[g], cuts[g])) return rc;
  }
  return 0;
}

// The stats of a device score call run in groups: `total` of its groups, whose `ran` groups that launched kernels
// left their counters, events and device plans' counts for collect().
void finish_groups(uis_model* m, const uis_stats& total, int jobs, int ran) {
  m->stats = total;
  m->last_U = jobs;
  m->last_groups = ran;
  m->stats_pending = ran > 0;
}

// Utterances [u0, u0 + U) of a host score call of U_all utterances: offsets `off` and labels `lab` rebased to the
// group, chains `cp`.  Staged, scored and copied back on their own: totals to scores_out[c][u0 + u] (scores_out points
// at column u0 of the call's [C][U_all]), increments to frame_out[u][c][..].  Leaves the group's stats in m->stats.
int score_host_group(uis_model* m, const double* const* seqs, int U, const int64_t* off, const int32_t* lab,
                     const ChainPlan& cp, float* scores_out, float* const* frame_out, int U_all, cudaStream_t st,
                     const DecodeParams& dp) {
  const int C = dp.count;
  const long long rows = off[U];
  begin_score_stats(m, U * C, rows, cp, st);
  if (rows == 0) return 0;  // (the totals are 0 already)
  int n_chunks = 0;
  bool staged = false;
  if (int rc = stage_host_rows(m, seqs, U, off, (size_t)rows, st, &n_chunks, &staged)) return rc;
  if (int rc = m->labels.ensure((size_t)rows * 4)) return rc;
  CU(cudaMemcpyAsync(m->labels.p, lab, (size_t)rows * 4, cudaMemcpyHostToDevice, st));
  if (int rc = m->sc_out.ensure(((size_t)U + (frame_out ? (size_t)rows : 0)) * C * 4)) return rc;
  float* dev_frames = frame_out ? m->sc_out.as<float>() + (size_t)U * C : nullptr;
  if (int rc = run_score(m, m->x32.as<float>(), off, U, &cp, m->labels.as<int32_t>(), m->sc_out.as<float>(),
                         dev_frames, st, /*gi_ready=*/true, dp))
    return rc;
  m->stats.kernel_launches += 2 * (int64_t)n_chunks;
  m->stats.chunks = n_chunks;
  m->stats.staged = staged ? 1 : 0;
  CU(cudaMemcpy2DAsync(scores_out, (size_t)U_all * 4, m->sc_out.p, (size_t)U * 4, (size_t)U * 4, C,
                       cudaMemcpyDeviceToHost, st));
  if (frame_out) {
    std::vector<float> inc((size_t)rows * C);
    CU(cudaMemcpyAsync(inc.data(), dev_frames, (size_t)rows * C * 4, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    for (int c = 0; c < C; ++c)  // config c's increments -> row c of the caller's [C][n] buffers
      for (int u = 0; u < U; ++u)
        if (off[u + 1] > off[u])
          std::memcpy(frame_out[u] + (size_t)c * (off[u + 1] - off[u]), inc.data() + (size_t)c * rows + off[u],
                      (size_t)(off[u + 1] - off[u]) * 4);
  }
  CU(cudaStreamSynchronize(st));
  if (int rc = collect(m)) return rc;
  CU(cudaEventElapsedTime(&m->stats.h2d_ms, m->ev_h2d[0], m->ev_h2d[1]));
  CU(cudaEventElapsedTime(&m->stats.pipeline_ms, m->ev_pipe, m->ev[1]));
  return 0;
}

int score_host_impl(uis_model* m, const double* const* seqs, const int64_t* n_frames, int U,
                    const int32_t* const* labels, float* scores_out, float* const* frame_out, cudaStream_t st,
                    const DecodeParams& dp) {
  const int C = dp.count;
  const auto t_begin = std::chrono::steady_clock::now();
  std::vector<int64_t> off(U + 1, 0);
  for (int u = 0; u < U; ++u) {
    if (n_frames[u] < 0) return fail(UIS_ERR_INVALID, "utterance %d: negative length", u);
    if (n_frames[u] > 0 && (!seqs[u] || !labels[u] || (frame_out && !frame_out[u])))
      return fail(UIS_ERR_INVALID, "utterance %d: null buffer", u);
    off[u + 1] = off[u] + n_frames[u];
  }
  const long long rows = off[U];
  std::vector<int32_t> lab((size_t)rows);
  for (int u = 0; u < U; ++u)
    if (n_frames[u] > 0) std::memcpy(lab.data() + off[u], labels[u], (size_t)n_frames[u] * 4);
  // Memory: per frame the score workspace, the staged fp32 rows, the labels and the per-frame outputs when asked
  size_t held = 0;
  const size_t per_row = score_row_bytes(m, true, &held) + 4 + (frame_out ? (size_t)4 * C : 0);
  held += m->labels.cap + m->sc_out.cap + m->x64.cap;
  const size_t fixed = score_fixed_bytes(m, U, C) +
                       (size_t)uis_model::kSlots * staging_chunk_rows(m->D_user) * m->D_user * 8;
  size_t max_rows = 0;
  if (rows > 0)
    if (int rc = row_budget(per_row, fixed, held, &max_rows)) return rc;
  const std::vector<int> cuts = rows > 0 ? cut_groups(off.data(), U, max_rows) : std::vector<int>{0, U};
  std::vector<ChainPlan> plans;
  if (int rc = plan_groups(lab.data(), off.data(), cuts, &plans)) return rc;
  std::fill(scores_out, scores_out + (size_t)U * C, 0.f);  // empty utterances score 0
  const int G = (int)plans.size();
  uis_stats total{};
  for (int g = 0; g < G; ++g) {
    const int u0 = cuts[g], u1 = cuts[g + 1];
    const std::vector<int64_t> goff = group_offsets(off.data(), u0, u1);
    if (int rc = score_host_group(m, seqs + u0, u1 - u0, goff.data(), lab.data() + off[u0], plans[g], scores_out + u0,
                                  frame_out ? frame_out + u0 : nullptr, U, st, dp))
      return rc;
    add_stats(&total, m->stats);
  }
  if (G > 1) m->stats = total;
  if (rows > 0) m->stats.host_ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t_begin).count();
  return 0;
}

int score_host(uis_model* m, const double* const* seqs, const int64_t* n_frames, int U, const int32_t* const* labels,
               float* scores_out, float* const* frame_out, void* stream, const DecodeParams& dp) {
  if (U < 0 || (U > 0 && (!seqs || !n_frames || !labels || !scores_out))) return fail(UIS_ERR_INVALID, "null argument");
  uis::DeviceGuard device_guard_(m->device);
  CU(device_guard_.status);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  CallOrder order(m, st);
  CU(order.status);
  const int rc = score_host_impl(m, seqs, n_frames, U, labels, scores_out, frame_out, st, dp);
  if (rc != 0 && rc != UIS_ERR_INVALID) drain_after_failure(m, st);
  return rc;
}

// A device-buffer score call in the groups `cuts` (cut_groups), one after the other on `st`.  Group [u0, u1) reads
// rows off[u0].. of x_dev (padded into the handle's x32 for a padded model: 16-byte aligned either way, as in
// predict_device_groups), labels_dev and ids_dev, and its reduce kernels write columns u0.. of the caller's [C][U]
// totals and [C][rows] increments in place (ScoreParams' row strides).  ids_dev: the chains are planned on the device,
// group by group, with nothing read back (each group's counts in its own slot of sc_counts); else `lab` holds the
// canonical labels of every row, read back by the caller, and the chains are planned here.
int score_device_groups(uis_model* m, const float* x_dev, const int64_t* off, int U, const std::vector<int32_t>& lab,
                        const int32_t* labels_dev, float* scores_dev, float* frame_dev, cudaStream_t st,
                        const DecodeParams& dp, const std::vector<int>& cuts, const int64_t* ids_dev = nullptr,
                        int32_t* labels_out = nullptr) {
  const int C = dp.count, G = (int)cuts.size() - 1;
  const long long rows = off[U];
  std::vector<ChainPlan> plans;
  if (!ids_dev)
    if (int rc = plan_groups(lab.data(), off, cuts, &plans)) return rc;
  // the handle's buffers, sized for the largest group before the first is enqueued: growing one later would free it
  // under the groups still in flight, which waits for them
  long long max_rows = 0;
  int max_u = 0;
  size_t plan_bytes = 0;
  for (int g = 0; g < G; ++g) {
    const long long r = off[cuts[g + 1]] - off[cuts[g]];
    max_rows = std::max(max_rows, r);
    max_u = std::max(max_u, cuts[g + 1] - cuts[g]);
    if (ids_dev && r > 0) plan_bytes = std::max(plan_bytes, uis::score_plan_bytes(r, cuts[g + 1] - cuts[g]));
  }
  const size_t R = (size_t)max_rows;
  if (int rc = m->gi.ensure(R * 3 * m->H * sizeof(float))) return rc;
  if (int rc = m->sc_mse.ensure(R * sizeof(float))) return rc;
  if (int rc = m->sc_blocks.ensure(R * sizeof(int))) return rc;
  if (int rc = m->row_off.ensure((size_t)(max_u + 1) * sizeof(long long))) return rc;
  if (m->D != m->D_user)
    if (int rc = m->x32.ensure(R * m->D * 4)) return rc;
  if (ids_dev) {
    if (int rc = m->labels.ensure(R * 4)) return rc;
    if (int rc = m->sc_chain_off.ensure((R + 1) * sizeof(long long))) return rc;
    if (int rc = m->sc_chain_rows.ensure(R * sizeof(long long))) return rc;
    if (int rc = m->sc_counts.ensure((size_t)4 * G * sizeof(int))) return rc;
    if (int rc = m->sc_plan.ensure(plan_bytes)) return rc;
  }
  uis_stats total{};
  int ran = 0;
  for (int g = 0; g < G; ++g) {
    const int u0 = cuts[g], u1 = cuts[g + 1], Ug = u1 - u0;
    const std::vector<int64_t> goff = group_offsets(off, u0, u1);
    const long long rg = goff[Ug];
    begin_score_stats(m, Ug * C, rg, ids_dev ? ChainPlan{} : plans[g], st);
    if (rg == 0) {  // empty utterances score 0
      CU(cudaMemset2DAsync(scores_dev + u0, (size_t)U * 4, 0, (size_t)Ug * 4, C, st));
      add_stats(&total, m->stats);
      continue;
    }
    const float* gx = x_dev + (size_t)off[u0] * m->D_user;
    if (int rc = pad_to_kernel_d(m, &gx, (size_t)rg, st)) return rc;
    float* gframe = frame_dev ? frame_dev + off[u0] : nullptr;
    const Group grp{ran, 0, rows, U};
    if (ids_dev) {
      std::vector<long long> off_ll(goff.begin(), goff.end());
      CU(cudaMemcpyAsync(m->row_off.p, off_ll.data(), (Ug + 1) * sizeof(long long), cudaMemcpyHostToDevice, st));
      CU(uis::score_plan(reinterpret_cast<const long long*>(ids_dev + off[u0]), m->row_off.as<long long>(), Ug, rg,
                         m->sc_plan.p, m->sc_plan.cap, m->labels.as<int>(), labels_out ? labels_out + off[u0] : nullptr,
                         m->sc_chain_off.as<long long>(), m->sc_chain_rows.as<long long>(),
                         m->sc_counts.as<int>() + 4 * ran, m->num_sms, st));
      m->last_score_counts = true;
      if (int rc = run_score(m, gx, goff.data(), Ug, nullptr, m->labels.as<int32_t>(), scores_dev + u0, gframe, st,
                             /*gi_ready=*/false, dp, grp))
        return rc;
      m->stats.kernel_launches += uis::kScorePlanLaunches;
    } else if (int rc = run_score(m, gx, goff.data(), Ug, &plans[g], labels_dev + off[u0], scores_dev + u0, gframe, st,
                                  /*gi_ready=*/false, dp, grp)) {
      return rc;
    }
    ++ran;
    add_stats(&total, m->stats);
  }
  finish_groups(m, total, U * C, ran);
  m->last_score_counts = ids_dev != nullptr;  // (an empty group's begin_score_stats cleared it)
  return 0;
}

int score_device(uis_model* m, const float* x_dev, const int64_t* frame_offsets, int U, const int32_t* labels_dev,
                 float* scores_dev, float* frame_dev, void* stream, const DecodeParams& dp) {
  if (U < 0 || (U > 0 && (!frame_offsets || !scores_dev))) return fail(UIS_ERR_INVALID, "null argument");
  for (int u = 0; u < U; ++u)
    if (frame_offsets[u + 1] < frame_offsets[u]) return fail(UIS_ERR_INVALID, "frame_offsets not monotone");
  const long long rows = U > 0 ? frame_offsets[U] : 0;
  if (rows > 0 && (!x_dev || !labels_dev)) return fail(UIS_ERR_INVALID, "null device buffer");
  uis::DeviceGuard device_guard_(m->device);
  CU(device_guard_.status);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  CallOrder order(m, st);
  CU(order.status);
  // the chain plan is made on the host: the labels come back first (this synchronises `stream`)
  std::vector<int32_t> lab((size_t)std::max(rows, 0ll));
  if (rows > 0) {
    CU(cudaMemcpyAsync(lab.data(), labels_dev, (size_t)rows * 4, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
  }
  size_t held = 0, max_rows = 0;
  const size_t per_row = score_row_bytes(m, m->D != m->D_user, &held);
  if (rows > 0)
    if (int rc = row_budget(per_row, score_fixed_bytes(m, U, dp.count), held, &max_rows)) return rc;
  const std::vector<int> cuts = rows > 0 ? cut_groups(frame_offsets, U, max_rows) : std::vector<int>{0, U};
  if (cuts.size() > 2) return score_device_groups(m, x_dev, frame_offsets, U, lab, labels_dev, scores_dev, frame_dev, st, dp, cuts);
  ChainPlan cp;
  if (int rc = plan_chains(lab.data(), frame_offsets, U, &cp)) return rc;
  begin_score_stats(m, U * dp.count, rows, cp, st);
  if (U == 0) return 0;
  if (rows == 0) {
    CU(cudaMemsetAsync(scores_dev, 0, (size_t)U * dp.count * 4, st));  // empty utterances score 0
    return 0;
  }
  if (int rc = pad_to_kernel_d(m, &x_dev, (size_t)rows, st)) return rc;
  return run_score(m, x_dev, frame_offsets, U, &cp, labels_dev, scores_dev, frame_dev, st, /*gi_ready=*/false, dp);
}

// score_device with arbitrary int64 ids per frame: the renaming and the chain plan run on the device (score_plan), so
// nothing is read back and the call only enqueues.
// The arguments are checked before the handle, so that a bad call is rejected the same way with or without a device.
int score_device_ids(uis_model* m, const float* x_dev, const int64_t* frame_offsets, int U, const int64_t* ids_dev,
                     float* scores_dev, float* frame_dev, int32_t* labels_dev, void* stream,
                     const uis_decode_params* params) {
  if (U < 0 || (U > 0 && (!frame_offsets || !scores_dev))) return fail(UIS_ERR_INVALID, "null argument");
  if (U > 0 && frame_offsets[0] != 0) return fail(UIS_ERR_INVALID, "frame_offsets[0] must be 0");
  for (int u = 0; u < U; ++u)
    if (frame_offsets[u + 1] < frame_offsets[u]) return fail(UIS_ERR_INVALID, "frame_offsets not monotone");
  const long long rows = U > 0 ? frame_offsets[U] : 0;
  if (rows > 0 && (!x_dev || !ids_dev)) return fail(UIS_ERR_INVALID, "null device buffer");
  // the input projection reads the rows with float4 loads; the ids are read as int64
  if (rows > 0 && (reinterpret_cast<uintptr_t>(x_dev) % 16 || reinterpret_cast<uintptr_t>(ids_dev) % 8))
    return fail(UIS_ERR_INVALID, "x_dev must be 16-byte aligned and ids_dev 8-byte aligned");
  if (rows >= 0x7fffffffll) return fail(UIS_ERR_UNSUPPORTED, "%lld frames: a device-planned score call holds < 2^31 - 1", rows);
  if (!m) return fail(UIS_ERR_INVALID, "model is NULL");
  DecodeParams dp;
  if (int rc = check_decode(params, U, &dp)) return rc;
  uis::DeviceGuard device_guard_(m->device);
  CU(device_guard_.status);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  CallOrder order(m, st);
  CU(order.status);
  if (rows > 0) {  // per frame: the score workspace, the canonical labels and the device plan's scratch
    size_t held = 0, max_rows = 0;
    const size_t per_row = score_row_bytes(m, m->D != m->D_user, &held) + 4 + uis::score_plan_bytes(rows, U) / (size_t)rows + 1;
    held += m->labels.cap + m->sc_plan.cap;
    if (int rc = row_budget(per_row, score_fixed_bytes(m, U, dp.count), held, &max_rows)) return rc;
    const std::vector<int> cuts = cut_groups(frame_offsets, U, max_rows);
    if (cuts.size() > 2)
      return score_device_groups(m, x_dev, frame_offsets, U, {}, nullptr, scores_dev, frame_dev, st, dp, cuts, ids_dev,
                                 labels_dev);
  }
  begin_score_stats(m, U * dp.count, rows, ChainPlan{}, st);
  if (U == 0) return 0;
  if (rows == 0) {
    CU(cudaMemsetAsync(scores_dev, 0, (size_t)U * dp.count * 4, st));  // empty utterances score 0
    return 0;
  }
  if (int rc = pad_to_kernel_d(m, &x_dev, (size_t)rows, st)) return rc;
  const size_t plan_bytes = uis::score_plan_bytes(rows, U);
  if (int rc = m->row_off.ensure((U + 1) * sizeof(long long))) return rc;
  if (int rc = m->labels.ensure((size_t)rows * 4)) return rc;
  if (int rc = m->sc_chain_off.ensure((size_t)(rows + 1) * sizeof(long long))) return rc;
  if (int rc = m->sc_chain_rows.ensure((size_t)rows * sizeof(long long))) return rc;
  if (int rc = m->sc_counts.ensure(4 * sizeof(int))) return rc;
  if (int rc = m->sc_plan.ensure(plan_bytes)) return rc;
  std::vector<long long> off_ll(frame_offsets, frame_offsets + U + 1);
  CU(cudaMemcpyAsync(m->row_off.p, off_ll.data(), (U + 1) * sizeof(long long), cudaMemcpyHostToDevice, st));
  CU(uis::score_plan(reinterpret_cast<const long long*>(ids_dev), m->row_off.as<long long>(), U, rows, m->sc_plan.p,
                     m->sc_plan.cap, m->labels.as<int>(), labels_dev, m->sc_chain_off.as<long long>(),
                     m->sc_chain_rows.as<long long>(), m->sc_counts.as<int>(), m->num_sms, st));
  m->last_score_counts = true;
  if (int rc = run_score(m, x_dev, frame_offsets, U, nullptr, m->labels.as<int32_t>(), scores_dev, frame_dev, st,
                         /*gi_ready=*/false, dp))
    return rc;
  m->stats.kernel_launches += uis::kScorePlanLaunches;
  return 0;
}

}  // namespace

extern "C" {

int uis_version(void) { return UIS_ABI_VERSION; }
const char* uis_last_error(void) { return g_err.c_str(); }

// Any (hidden <= 1024, dim <= 512) runs in the smallest instantiated kernel shape that holds it, zero-padded: a padded
// hidden unit has zero weights and biases (r = z = 1/2, n = 0, so it stays at its initial 0) and feeds nothing; a
// padded observation dimension has x = mean = 0 and adds (0 - 0)^2 * w = 0 to every Gaussian term.  Adding exact
// zeros does not change an fp32 sum, so the results are those of a kernel instantiated for the caller's shape.
int uis_model_create(uis_model** out, int device, int D, int H, int depth, const float* w_ih, const float* w_hh,
                     const float* b_ih, const float* b_hh, const float* w1, const float* b1, const float* w2,
                     const float* b2, const float* h0, const float* sigma2, double transition_bias,
                     double crp_alpha) {
  if (!out) return fail(UIS_ERR_INVALID, "out is NULL");
  *out = nullptr;
  if (!w_ih || !w_hh || !b_ih || !b_hh || !w1 || !b1 || !w2 || !b2 || !h0 || !sigma2)
    return fail(UIS_ERR_INVALID, "NULL weight pointer");
  if (depth < 1 || depth > uis::kMaxDepth)
    return fail(UIS_ERR_UNSUPPORTED, "rnn_depth=%d: the sm_90a kernels support 1..%d stacked GRU layers", depth, uis::kMaxDepth);
  if (D < 1 || H < 1) return fail(UIS_ERR_INVALID, "observation_dim and rnn_hidden_size must be >= 1");
  int Hp = 0, Dp = 0;
  for (auto& sh : uis::kShapes)
    if (!Hp && H <= sh[0] && D <= sh[1]) { Hp = sh[0]; Dp = sh[1]; }
  if (!Hp)
    return fail(UIS_ERR_UNSUPPORTED, "hidden=%d dim=%d: the sm_90a kernels hold models up to hidden=1024 dim=512", H, D);
  if (Hp == H && Dp == D)
    return model_create_impl(out, device, D, H, depth, w_ih, w_hh, b_ih, b_hh, w1, b1, w2, b2, h0, sigma2,
                             transition_bias, crp_alpha, D, H);
  uis::DeviceGuard device_guard_(device);
  CU(device_guard_.status);
  std::vector<float> v, p_wih((size_t)3 * Hp * Dp + (size_t)(depth - 1) * 3 * Hp * Hp, 0.f), p_whh((size_t)depth * 3 * Hp * Hp, 0.f),
      p_bih((size_t)depth * 3 * Hp, 0.f), p_bhh((size_t)depth * 3 * Hp, 0.f), p_w1((size_t)Hp * Hp, 0.f), p_b1(Hp, 0.f),
      p_w2((size_t)Dp * Hp, 0.f), p_b2(Dp, 0.f), p_h0((size_t)depth * Hp, 0.f), p_s2(Dp, 1.f);
  // gate blocks (r, z, n) keep their own row ranges: row g * H + j -> g * Hp + j
  if (int r = fetch(v, w_ih, (size_t)3 * H * D + (size_t)(depth - 1) * 3 * H * H)) return r;
  for (int g = 0; g < 3; ++g)
    for (int j = 0; j < H; ++j)
      std::copy(v.begin() + ((size_t)g * H + j) * D, v.begin() + ((size_t)g * H + j + 1) * D,
                p_wih.begin() + ((size_t)g * Hp + j) * Dp);
  for (int l = 1; l < depth; ++l)
    for (int g = 0; g < 3; ++g)
      for (int j = 0; j < H; ++j) {
        const float* src = v.data() + (size_t)3 * H * D + (size_t)(l - 1) * 3 * H * H + ((size_t)g * H + j) * H;
        std::copy(src, src + H, p_wih.begin() + (size_t)3 * Hp * Dp + (size_t)(l - 1) * 3 * Hp * Hp + ((size_t)g * Hp + j) * Hp);
      }
  if (int r = fetch(v, w_hh, (size_t)depth * 3 * H * H)) return r;
  for (int l = 0; l < depth; ++l)
    for (int g = 0; g < 3; ++g)
      for (int j = 0; j < H; ++j) {
        const float* src = v.data() + (size_t)l * 3 * H * H + ((size_t)g * H + j) * H;
        std::copy(src, src + H, p_whh.begin() + (size_t)l * 3 * Hp * Hp + ((size_t)g * Hp + j) * Hp);
      }
  for (int which = 0; which < 2; ++which) {
    if (int r = fetch(v, which ? b_hh : b_ih, (size_t)depth * 3 * H)) return r;
    std::vector<float>& dst = which ? p_bhh : p_bih;
    for (int l = 0; l < depth; ++l)
      for (int g = 0; g < 3; ++g)
        std::copy(v.begin() + ((size_t)l * 3 + g) * H, v.begin() + ((size_t)l * 3 + g + 1) * H,
                  dst.begin() + ((size_t)l * 3 + g) * Hp);
  }
  if (int r = fetch(v, w1, (size_t)H * H)) return r;
  for (int j = 0; j < H; ++j) std::copy(v.begin() + (size_t)j * H, v.begin() + (size_t)(j + 1) * H, p_w1.begin() + (size_t)j * Hp);
  if (int r = fetch(v, b1, H)) return r;
  std::copy(v.begin(), v.end(), p_b1.begin());
  if (int r = fetch(v, w2, (size_t)D * H)) return r;
  for (int d = 0; d < D; ++d) std::copy(v.begin() + (size_t)d * H, v.begin() + (size_t)(d + 1) * H, p_w2.begin() + (size_t)d * Hp);
  if (int r = fetch(v, b2, D)) return r;
  std::copy(v.begin(), v.end(), p_b2.begin());
  if (int r = fetch(v, h0, (size_t)depth * H)) return r;
  for (int l = 0; l < depth; ++l) std::copy(v.begin() + (size_t)l * H, v.begin() + (size_t)(l + 1) * H, p_h0.begin() + (size_t)l * Hp);
  if (int r = fetch(v, sigma2, D)) return r;
  std::copy(v.begin(), v.end(), p_s2.begin());
  return model_create_impl(out, device, Dp, Hp, depth, p_wih.data(), p_whh.data(), p_bih.data(), p_bhh.data(), p_w1.data(),
                           p_b1.data(), p_w2.data(), p_b2.data(), p_h0.data(), p_s2.data(), transition_bias, crp_alpha, D, H);
}

int uis_model_destroy(uis_model* m) {
  if (!m) return 0;
  uis::DeviceGuard device_guard_(m->device);
  DevBuf* bufs[] = {&m->wih_t, &m->whh_t, &m->w1_t, &m->w2_t, &m->bih, &m->bhh, &m->b1, &m->b2, &m->wvec, &m->mean0,
                    &m->hidden0, &m->wih_up_t, &m->logn, &m->own_logs.tot, &m->own_logs.cfg, &m->sweep_logs.tot, &m->sweep_logs.cfg, &m->x64, &m->x32, &m->gi, &m->row_off, &m->order,
                    &m->pool_mean, &m->pool_hidden, &m->bp, &m->queue_stats, &m->labels, &m->status, &m->dbg_win,
                    &m->dbg_score, &m->dbg_off, &m->dbg_final_scores, &m->dbg_final_k, &m->dbg_best_mean,
                    &m->dbg_best_hidden, &m->dbg_best_blocks, &m->tc_planes, &m->tc_scratch, &m->pool_mse, &m->stat_bar, &m->stat_scratch,
                    &m->tree_arena, &m->nb_scores, &m->nb_speakers, &m->nb_count, &m->sc_chain_off,
                    &m->sc_chain_rows, &m->sc_mse, &m->sc_blocks, &m->sc_out, &m->sc_counts, &m->sc_plan};
  for (DevBuf* b : bufs) b->release();
  for (auto& e : m->ev)
    if (e) cudaEventDestroy(e);
  for (auto& e : m->ev_copied)
    if (e) cudaEventDestroy(e);
  for (auto& e : m->ev_free)
    if (e) cudaEventDestroy(e);
  for (auto& e : m->ev_h2d)
    if (e) cudaEventDestroy(e);
  if (m->ev_pipe) cudaEventDestroy(m->ev_pipe);
  if (m->ev_done) cudaEventDestroy(m->ev_done);
  if (m->copy_stream) cudaStreamDestroy(m->copy_stream);
  if (m->labels_pin) cudaFreeHost(m->labels_pin);
  for (auto& e : m->ev_dma)
    if (e) cudaEventDestroy(e);
  if (m->pin_stage) cudaFreeHost(m->pin_stage);
  delete m->copy_pool;
  delete m;
  return 0;
}

int uis_model_constants(uis_model* m, float* mean0, float* hidden0) {
  if (!m) return fail(UIS_ERR_INVALID, "model is NULL");
  uis::DeviceGuard device_guard_(m->device);
  CU(device_guard_.status);
  if (mean0) CU(cudaMemcpy(mean0, m->mean0.p, m->D_user * 4, cudaMemcpyDeviceToHost));
  if (hidden0)
    CU(cudaMemcpy2D(hidden0, (size_t)m->H_user * 4, m->hidden0.p, (size_t)m->H * 4, (size_t)m->H_user * 4, m->depth,
                    cudaMemcpyDeviceToHost));
  return 0;
}

size_t uis_predict_workspace_bytes(uis_model* m, const int64_t* frame_offsets, int U, const uis_predict_opts* opts) {
  Plan pl;
  if (make_plan(m, frame_offsets, U, opts, &pl)) return 0;
  return workspace_bytes(m, pl, U);
}

int uis_predict_device(uis_model* m, const float* x_dev, const int64_t* frame_offsets, int U,
                       const uis_predict_opts* opts, int32_t* labels_dev, const uis_debug_taps* taps, void* stream) {
  return uis_predict_device_bounded(m, x_dev, frame_offsets, U, opts, labels_dev, taps, stream, nullptr, nullptr, nullptr);
}

int uis_predict_device_bounded(uis_model* m, const float* x_dev, const int64_t* frame_offsets, int U,
                               const uis_predict_opts* opts, int32_t* labels_dev, const uis_debug_taps* taps, void* stream,
                               const int32_t* max_speakers, const int32_t* min_speakers, int32_t* speakers_dev) {
  return predict_device_impl(m, x_dev, frame_offsets, U, opts, labels_dev, taps, stream, max_speakers, min_speakers,
                             speakers_dev, NBestOut{});
}

int uis_predict_device_nbest(uis_model* m, const float* x_dev, const int64_t* frame_offsets, int U,
                             const uis_predict_opts* opts, const uis_debug_taps* taps, void* stream,
                             const int32_t* max_speakers, const int32_t* min_speakers, int32_t n_best,
                             const uis_nbest_out* out) {
  if (!opts || !out) return fail(UIS_ERR_INVALID, "null argument");
  if (int rc = check_nbest(n_best, opts, out)) return rc;
  return predict_device_impl(m, x_dev, frame_offsets, U, opts, out->labels_dev, taps, stream, max_speakers, min_speakers,
                             nullptr, NBestOut{n_best, out->scores, out->speakers, out->count});
}

int uis_predict_device_sweep(uis_model* m, const float* x_dev, const int64_t* frame_offsets, int U,
                             const uis_predict_opts* opts, const uis_debug_taps* taps, void* stream,
                             const int32_t* max_speakers, const int32_t* min_speakers, int32_t n_best,
                             const uis_nbest_out* out, const uis_decode_params* params) {
  if (!m || !opts || !out) return fail(UIS_ERR_INVALID, "null argument");
  if (int rc = check_nbest(n_best, opts, out)) return rc;
  DecodeParams dp;
  if (int rc = check_decode(params, U, &dp)) return rc;
  return predict_device_impl(m, x_dev, frame_offsets, U, opts, out->labels_dev, taps, stream, max_speakers, min_speakers,
                             nullptr, NBestOut{n_best, out->scores, out->speakers, out->count}, &dp);
}

int uis_predict(uis_model* m, const double* const* seqs, const int64_t* n_frames, int U, const uis_predict_opts* opts,
                int32_t* const* labels_out, const uis_debug_taps* taps, void* stream) {
  return uis_predict_bounded(m, seqs, n_frames, U, opts, labels_out, taps, stream, nullptr, nullptr, nullptr);
}

int uis_predict_bounded(uis_model* m, const double* const* seqs, const int64_t* n_frames, int U,
                        const uis_predict_opts* opts, int32_t* const* labels_out, const uis_debug_taps* taps, void* stream,
                        const int32_t* max_speakers, const int32_t* min_speakers, int32_t* speakers_out) {
  return predict_host_impl(m, seqs, n_frames, U, opts, labels_out, taps, stream, max_speakers, min_speakers,
                           speakers_out, NBestOut{});
}

int uis_predict_nbest(uis_model* m, const double* const* seqs, const int64_t* n_frames, int U,
                      const uis_predict_opts* opts, const uis_debug_taps* taps, void* stream,
                      const int32_t* max_speakers, const int32_t* min_speakers, int32_t n_best,
                      const uis_nbest_out* out) {
  if (!opts || !out) return fail(UIS_ERR_INVALID, "null argument");
  if (int rc = check_nbest(n_best, opts, out)) return rc;
  return predict_host_impl(m, seqs, n_frames, U, opts, out->labels_out, taps, stream, max_speakers, min_speakers,
                           nullptr, NBestOut{n_best, out->scores, out->speakers, out->count});
}

int uis_predict_sweep(uis_model* m, const double* const* seqs, const int64_t* n_frames, int U,
                      const uis_predict_opts* opts, const uis_debug_taps* taps, void* stream,
                      const int32_t* max_speakers, const int32_t* min_speakers, int32_t n_best,
                      const uis_nbest_out* out, const uis_decode_params* params) {
  if (!m || !opts || !out) return fail(UIS_ERR_INVALID, "null argument");
  if (int rc = check_nbest(n_best, opts, out)) return rc;
  DecodeParams dp;
  if (int rc = check_decode(params, U, &dp)) return rc;
  return predict_host_impl(m, seqs, n_frames, U, opts, out->labels_out, taps, stream, max_speakers, min_speakers,
                           nullptr, NBestOut{n_best, out->scores, out->speakers, out->count}, &dp);
}

int uis_get_stats(uis_model* m, uis_stats* out) {
  if (!m || !out) return fail(UIS_ERR_INVALID, "null argument");
  uis::DeviceGuard device_guard_(m->device);
  CU(device_guard_.status);
  const int rc = collect(m);
  *out = m->stats;
  return rc;
}

int uis_score(uis_model* m, const double* const* seqs, const int64_t* n_frames, int U, const int32_t* const* labels,
              float* scores_out, float* const* frame_out, void* stream) {
  if (!m) return fail(UIS_ERR_INVALID, "model is NULL");
  return score_host(m, seqs, n_frames, U, labels, scores_out, frame_out, stream, model_decode(m));
}

int uis_score_sweep(uis_model* m, const double* const* seqs, const int64_t* n_frames, int U, const int32_t* const* labels,
                    float* scores_out, float* const* frame_out, void* stream, const uis_decode_params* params) {
  if (!m) return fail(UIS_ERR_INVALID, "model is NULL");
  DecodeParams dp;
  if (int rc = check_decode(params, U, &dp)) return rc;
  return score_host(m, seqs, n_frames, U, labels, scores_out, frame_out, stream, dp);
}

int uis_score_device(uis_model* m, const float* x_dev, const int64_t* frame_offsets, int U, const int32_t* labels_dev,
                     float* scores_dev, float* frame_dev, void* stream) {
  if (!m) return fail(UIS_ERR_INVALID, "model is NULL");
  return score_device(m, x_dev, frame_offsets, U, labels_dev, scores_dev, frame_dev, stream, model_decode(m));
}

int uis_score_device_sweep(uis_model* m, const float* x_dev, const int64_t* frame_offsets, int U,
                           const int32_t* labels_dev, float* scores_dev, float* frame_dev, void* stream,
                           const uis_decode_params* params) {
  if (!m) return fail(UIS_ERR_INVALID, "model is NULL");
  DecodeParams dp;
  if (int rc = check_decode(params, U, &dp)) return rc;
  return score_device(m, x_dev, frame_offsets, U, labels_dev, scores_dev, frame_dev, stream, dp);
}

int uis_score_device_ids(uis_model* m, const float* x_dev, const int64_t* frame_offsets, int U, const int64_t* ids_dev,
                         float* scores_dev, float* frame_dev, int32_t* labels_dev, void* stream,
                         const uis_decode_params* params) {
  return score_device_ids(m, x_dev, frame_offsets, U, ids_dev, scores_dev, frame_dev, labels_dev, stream, params);
}

}  // extern "C"
