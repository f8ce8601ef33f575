// fit() on the device: one training iteration of UISRNN.fit_concatenated
// (reference uisrnn/uisrnn.py:252-295) as hand-written sm_90a kernels behind a C ABI:
//   packed-sequence GRU forward (:262-263 -> CoreRNN.forward :45-52), MLP, running mean over time
//   (:265-271), masked weighted-MSE likelihood (:274-277, loss_func.py:19-41), sigma^2 prior
//   (:280-284, loss_func.py:44-60), parameter-norm regulariser (:287-288, loss_func.py:63-76),
//   full backward pass (what autograd does at :290), gradient-norm clipping of the RNN parameters
//   (:292), Adam step (:293, torch.optim.Adam defaults) and the sigma^2 clamp (:295).
// Layout: time-major zero-padded batch X[L][B][D] with per-sequence lengths sorted descending
// (exactly what utils.pack_sequence builds before pack_padded_sequence, utils.py:237-246); at time
// t the first batch_t = #{len_b > t} sequences are live, as in a PackedSequence.
// All arithmetic fp32.  The derivation of the backward pass is checked against torch autograd in
// tools/fit_manual_check.py (CPU) and tests/test_gpu_fit.py (device).
#include <cooperative_groups.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/uisrnn_b200.h"
#include "uis_common.cuh"

namespace uis {
int api_fail(int code, const char* fmt, ...);  // defined in uis_api.cu (sets uis_last_error)
}

#define CUT(call)                                                                                   \
  do {                                                                                              \
    cudaError_t e_ = (call);                                                                        \
    if (e_ != cudaSuccess)                                                                          \
      return uis::api_fail(UIS_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
  } while (0)

namespace uis {

// ---------------------------------------------------------------------------------------------
// Generic fp32 GEMM:  C[M][N] (+)= opA(A)[M][K] * opB(B)[K][N]  (+ bias[N]) (relu) (* (mask > 0))
//   TA == false: A stored [M][K];  TA == true: A stored [K][M]
//   TB == false: B stored [K][N];  TB == true: B stored [N][K]   (PyTorch Linear weight layout)
// 64x64 CTA tile, BK = 16, 256 threads, 4x4 register micro-tile, k ascending per thread.
template <bool TA, bool TB>
__global__ void __launch_bounds__(256) gemm_kernel(const float* __restrict__ A, const float* __restrict__ B,
                                                   const float* __restrict__ bias, const float* __restrict__ mask,
                                                   float* __restrict__ C, int M, int N, int K, int relu,
                                                   int accumulate, float* __restrict__ partial,
                                                   unsigned* __restrict__ tickets) {
  __shared__ float As[16][64 + 1];
  __shared__ float Bs[16][64 + 1];
  __shared__ unsigned last_flag;
  const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;
  const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
  // split-K over gridDim.z (weight-gradient products have K = #rows in the thousands but few tiles)
  const int splits = gridDim.z;
  const int kslice = ((K + splits - 1) / splits + 15) / 16 * 16;
  const int kbeg = blockIdx.z * kslice, kend = min(K, kbeg + kslice);
  float acc[4][4] = {};
  for (int k0 = kbeg; k0 < kend; k0 += 16) {
    for (int q = tid; q < 64 * 16; q += 256) {
      int mm, kk;
      if (TA) { mm = q % 64; kk = q / 64; } else { kk = q % 16; mm = q / 16; }
      const int gm = m0 + mm, gk = k0 + kk;
      float v = 0.f;
      if (gm < M && gk < kend) v = TA ? A[(size_t)gk * M + gm] : A[(size_t)gm * K + gk];
      As[kk][mm] = v;
    }
    for (int q = tid; q < 64 * 16; q += 256) {
      int nn, kk;
      if (TB) { kk = q % 16; nn = q / 16; } else { nn = q % 64; kk = q / 64; }
      const int gn = n0 + nn, gk = k0 + kk;
      float v = 0.f;
      if (gn < N && gk < kend) v = TB ? B[(size_t)gn * K + gk] : B[(size_t)gk * N + gn];
      Bs[kk][nn] = v;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = As[kk][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = Bs[kk][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
  if (splits > 1) {  // park the partial tile; the last CTA of this tile folds all of them in order
    const unsigned tile_id = blockIdx.y * gridDim.x + blockIdx.x;
    float* mine = partial + ((size_t)tile_id * splits + blockIdx.z) * (64 * 64);
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) mine[(ty * 4 + i) * 64 + tx * 4 + j] = acc[i][j];
    __threadfence();
    __syncthreads();
    if (tid == 0) {
      const unsigned t = atomicAdd(&tickets[tile_id], 1u);
      last_flag = (t == (unsigned)splits - 1) ? 1u : 0u;
      if (last_flag) tickets[tile_id] = 0;
    }
    __syncthreads();
    if (!last_flag) return;
    __threadfence();
    const float* tile = partial + (size_t)tile_id * splits * (64 * 64);
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float v = 0.f;
        for (int s2 = 0; s2 < splits; ++s2) v += tile[(size_t)s2 * (64 * 64) + (ty * 4 + i) * 64 + tx * 4 + j];
        acc[i][j] = v;
      }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int gm = m0 + ty * 4 + i;
    if (gm >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int gn = n0 + tx * 4 + j;
      if (gn >= N) continue;
      float v = acc[i][j];
      if (bias) v += bias[gn];
      if (relu) v = fmaxf(v, 0.f);
      if (mask) v = (mask[(size_t)gm * N + gn] > 0.f) ? v : 0.f;
      if (accumulate) v += C[(size_t)gm * N + gn];
      C[(size_t)gm * N + gn] = v;
    }
  }
}

// The same product on 128x128 CTA tiles (BK = 16, 256 threads, 8x8 register micro-tile: rows ty*8.., columns tx*4.. and
// 64+tx*4..; operands of the inner loop come from shared memory as float4, broadcast over the half-warp for A and
// contiguous for B): 4x the flops per shared-memory byte of the 64x64 kernel.  Used when both M and N reach 128.
template <bool TA, bool TB>
__global__ void __launch_bounds__(256, 2) gemm128_kernel(const float* __restrict__ A, const float* __restrict__ B,
                                                      const float* __restrict__ bias, const float* __restrict__ mask,
                                                      float* __restrict__ C, int M, int N, int K, int relu,
                                                      int accumulate, float* __restrict__ partial,
                                                      unsigned* __restrict__ tickets) {
  __shared__ __align__(16) float As[16][128 + 4];
  __shared__ __align__(16) float Bs[16][128 + 4];
  __shared__ unsigned last_flag;
  const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;
  const int m0 = blockIdx.y * 128, n0 = blockIdx.x * 128;
  const int splits = gridDim.z;
  const int kslice = ((K + splits - 1) / splits + 15) / 16 * 16;
  const int kbeg = blockIdx.z * kslice, kend = min(K, kbeg + kslice);
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
  for (int k0 = kbeg; k0 < kend; k0 += 16) {
#pragma unroll
    for (int r = 0; r < 8; ++r) {  // 128 x 16 elements per operand, 8 per thread, coalesced along the stored-contiguous axis
      const int q = tid + r * 256;
      int mm, kk;
      if (TA) { mm = q % 128; kk = q / 128; } else { kk = q % 16; mm = q / 16; }
      const int gm = m0 + mm, gk = k0 + kk;
      float v = 0.f;
      if (gm < M && gk < kend) v = TA ? A[(size_t)gk * M + gm] : A[(size_t)gm * K + gk];
      As[kk][mm] = v;
    }
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const int q = tid + r * 256;
      int nn, kk;
      if (TB) { kk = q % 16; nn = q / 16; } else { nn = q % 128; kk = q / 128; }
      const int gn = n0 + nn, gk = k0 + kk;
      float v = 0.f;
      if (gn < N && gk < kend) v = TB ? B[(size_t)gn * K + gk] : B[(size_t)gk * N + gn];
      Bs[kk][nn] = v;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) {
      const float4 a0 = *reinterpret_cast<const float4*>(&As[kk][ty * 8]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[kk][ty * 8 + 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4*>(&Bs[kk][64 + tx * 4]);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
  // element (i, j) of the micro-tile -> tile coordinates
  auto row_of = [&](int i) { return ty * 8 + i; };
  auto col_of = [&](int j) { return (j < 4 ? 0 : 64) + tx * 4 + (j & 3); };
  if (splits > 1) {  // park the partial tile; the last CTA of this tile folds all of them in order
    const unsigned tile_id = blockIdx.y * gridDim.x + blockIdx.x;
    float* mine = partial + ((size_t)tile_id * splits + blockIdx.z) * (128 * 128);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      *reinterpret_cast<float4*>(mine + row_of(i) * 128 + col_of(0)) = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
      *reinterpret_cast<float4*>(mine + row_of(i) * 128 + col_of(4)) = make_float4(acc[i][4], acc[i][5], acc[i][6], acc[i][7]);
    }
    __threadfence();
    __syncthreads();
    if (tid == 0) {
      const unsigned t = atomicAdd(&tickets[tile_id], 1u);
      last_flag = (t == (unsigned)splits - 1) ? 1u : 0u;
      if (last_flag) tickets[tile_id] = 0;
    }
    __syncthreads();
    if (!last_flag) return;
    __threadfence();
    const float* tile = partial + (size_t)tile_id * splits * (128 * 128);
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int s2 = 0; s2 < splits; ++s2) {
          const float4 q = *reinterpret_cast<const float4*>(tile + (size_t)s2 * (128 * 128) + row_of(i) * 128 + col_of(4 * h));
          v.x += q.x; v.y += q.y; v.z += q.z; v.w += q.w;
        }
        acc[i][4 * h] = v.x; acc[i][4 * h + 1] = v.y; acc[i][4 * h + 2] = v.z; acc[i][4 * h + 3] = v.w;
      }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int gm = m0 + row_of(i);
    if (gm >= M) continue;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int gn = n0 + col_of(j);
      if (gn >= N) continue;
      float v = acc[i][j];
      if (bias) v += bias[gn];
      if (relu) v = fmaxf(v, 0.f);
      if (mask) v = (mask[(size_t)gm * N + gn] > 0.f) ? v : 0.f;
      if (accumulate) v += C[(size_t)gm * N + gn];
      C[(size_t)gm * N + gn] = v;
    }
  }
}

// column sums: out[n] = sum_r A[r][n].  grid (N / 32 column groups, row slices): every block sums its slice of the rows
// (8 warps striding over it) and the slices meet through a ticket: the LAST block of a column group adds the partial
// sums in slice order -- deterministic, one launch, and enough blocks to pull the matrix at HBM/L2 speed (the earlier
// one-block-per-column-group version took 29 us for a 3200 x 1536 matrix).
constexpr int kColsumSlices = 16;
__global__ void colsum_kernel(const float* __restrict__ A, float* __restrict__ out, int R, int N,
                              float* __restrict__ partial /*[N / 32 groups][slices][32]*/, unsigned* __restrict__ tickets) {
  __shared__ float part[8][32];
  __shared__ unsigned last_flag;
  const int lane = threadIdx.x % 32, w = threadIdx.x / 32;
  const int n = blockIdx.x * 32 + lane, S = gridDim.y;
  const int rows_per = (R + S - 1) / S, r0 = blockIdx.y * rows_per, r1 = min(R, r0 + rows_per);
  float s = 0.f;
  if (n < N)
    for (int r = r0 + w; r < r1; r += 8) s += A[(size_t)r * N + n];
  part[w][lane] = s;
  __syncthreads();
  if (w == 0) {
    float t = 0.f;
    for (int q = 0; q < 8; ++q) t += part[q][lane];
    if (S == 1) {
      if (n < N) out[n] = t;
    } else {
      partial[((size_t)blockIdx.x * S + blockIdx.y) * 32 + lane] = t;
    }
  }
  if (S == 1) return;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned tk = atomicAdd(&tickets[blockIdx.x], 1u);
    last_flag = (tk == (unsigned)S - 1) ? 1u : 0u;
    if (last_flag) tickets[blockIdx.x] = 0;
  }
  __syncthreads();
  if (!last_flag) return;
  __threadfence();
  if (w == 0 && n < N) {
    float t = 0.f;
    for (int q = 0; q < S; ++q) t += partial[((size_t)blockIdx.x * S + q) * 32 + lane];
    out[n] = t;
  }
}

// ---------------------------------------------------------------------------------------------
// Recurrent products of one time step:  C[b][n] (+)= sum_k A[b][k] * W[k][n],  b < nb <= 32.
// The output is only 32 rows tall, so parallelism comes from the K dimension: grid = (N/64 column
// tiles, kSplit K-slices).  Each CTA multiplies its 32 x 64 x (K/kSplit) slab with shared-memory
// tiles (coalesced loads), parks the partial tile in global memory, and the LAST CTA to finish a
// column tile (atomic ticket) adds the kSplit partials in a fixed order -- deterministic, one launch.
constexpr int kSplit = 16;
__global__ void __launch_bounds__(256) splitk_gemm_kernel(const float* __restrict__ A, int lda,
                                                          const float* __restrict__ W, float* __restrict__ C, int ldc,
                                                          int nb, int N, int K, int accumulate,
                                                          float* __restrict__ partial, unsigned* __restrict__ tickets) {
  __shared__ float As[16][32 + 1];
  __shared__ float Ws[16][64 + 1];
  __shared__ unsigned last_flag;
  const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;  // micro-tile: rows ty*2.., cols tx*4..
  const int n0 = blockIdx.x * 64, sp = blockIdx.y;
  const int kslice = ((K + kSplit - 1) / kSplit + 15) / 16 * 16;
  const int k0 = sp * kslice, k1 = min(K, k0 + kslice);
  float acc[2][4] = {};
  for (int kb = k0; kb < k1; kb += 16) {
    for (int q = tid; q < 32 * 16; q += 256) {
      const int kk = q % 16, b = q / 16;
      As[kk][b] = (b < nb && kb + kk < k1) ? A[(size_t)b * lda + kb + kk] : 0.f;
    }
    for (int q = tid; q < 64 * 16; q += 256) {
      const int nn = q % 64, kk = q / 64;
      Ws[kk][nn] = (n0 + nn < N && kb + kk < k1) ? W[(size_t)(kb + kk) * N + n0 + nn] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) {
      const float a0 = As[kk][ty * 2], a1 = As[kk][ty * 2 + 1];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float w = Ws[kk][tx * 4 + j];
        acc[0][j] = fmaf(a0, w, acc[0][j]);
        acc[1][j] = fmaf(a1, w, acc[1][j]);
      }
    }
    __syncthreads();
  }
  float* mine = partial + ((size_t)blockIdx.x * kSplit + sp) * (32 * 64);
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) mine[(ty * 2 + i) * 64 + tx * 4 + j] = acc[i][j];
  __threadfence();
  __syncthreads();
  if (tid == 0) {
    const unsigned t = atomicAdd(&tickets[blockIdx.x], 1u);
    last_flag = (t == kSplit - 1) ? 1u : 0u;
    if (last_flag) tickets[blockIdx.x] = 0;  // ready for the next launch
  }
  __syncthreads();
  if (!last_flag) return;
  __threadfence();
  const float* tile = partial + (size_t)blockIdx.x * kSplit * (32 * 64);
  for (int q = tid; q < 32 * 64; q += 256) {
    const int b = q / 64, nn = q % 64;
    if (b < nb && n0 + nn < N) {
      float v = 0.f;
#pragma unroll
      for (int s2 = 0; s2 < kSplit; ++s2) v += tile[(size_t)s2 * (32 * 64) + q];
      float* dst = C + (size_t)b * ldc + n0 + nn;
      *dst = accumulate ? (*dst + v) : v;
    }
  }
}

// GRU gates of one time step (PyTorch order r,z,n):  gh = W_hh h_{t-1} (no bias yet), b < nb
__global__ void gru_gate_fwd_kernel(const float* __restrict__ gh, const float* __restrict__ bhh,
                                    const float* __restrict__ gi_t, const float* __restrict__ hprev,
                                    float* __restrict__ hnew, float* __restrict__ r_t, float* __restrict__ z_t,
                                    float* __restrict__ n_t, float* __restrict__ hn_t, int nb, int H) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= nb * H) return;
  const int b = q / H, j = q % H;
  const float* g = gh + (size_t)b * 3 * H;
  const float* gi = gi_t + (size_t)b * 3 * H;
  const float r = sigmoid_f32(gi[j] + (g[j] + bhh[j]));
  const float z = sigmoid_f32(gi[H + j] + (g[H + j] + bhh[H + j]));
  const float hn = g[2 * H + j] + bhh[2 * H + j];
  const float n = tanhf(gi[2 * H + j] + r * hn);
  const float hp = hprev[q];
  hnew[q] = (hp - n) * z + n;
  r_t[q] = r; z_t[q] = z; n_t[q] = n; hn_t[q] = hn;
}

// ---------------------------------------------------------------------------------------------
// Persistent recurrence kernels (one cooperative launch per direction instead of two launches per time step).
// The sequential part of an iteration is L dependent products with W_hh (3 MB) on <= 32 rows: far too little
// work per step for a launch each (a launch + drain costs more than the step's arithmetic).  Here CTA c owns
// kUPC = 4 hidden units for the whole sequence -- the 12 rows (forward) / 4 columns (backward) of W_hh it
// needs stay in its shared memory (24 KB) for all L steps -- and the CTAs exchange h_t (forward) / dGh_t
// (backward) through L2 with one grid-wide barrier per step (cooperative_groups grid.sync(): the cooperative launch
// makes all CTAs co-resident).  H % 128 == 0, H / 4 CTAs (128 at H = 512).
constexpr int kUPC = 4;
// One launch covers a group of <= 32 batch columns [b0, b0 + B) of a batch that is `stride` columns wide (the
// pointers handed to the kernels are already offset to column b0); wider batches run group after group.
struct SeqParams { int length[32]; int L, B, H, stride; };

__device__ __forceinline__ int seq_rows_alive(const SeqParams& sp, int t) {
  int nb = 0;
  for (int b = 0; b < sp.B; ++b) nb += sp.length[b] > t ? 1 : 0;
  return nb;
}

// Forward: for t = 0..L-1, rows b < nb(t):  gh = W_hh h_{t-1};  (r, z, n, h_t) as gru_gate_fwd_kernel.
// hs: [(L+1)*B][H] with hs[0..B) = h_{-1};  gi: [L*B][3H] = W_ih x + b_ih.
__global__ void __launch_bounds__(256) gru_seq_fwd_kernel(const float* __restrict__ whh, const float* __restrict__ bhh,
                                                          const float* __restrict__ gi, float* hs,
                                                          float* __restrict__ r_o, float* __restrict__ z_o,
                                                          float* __restrict__ n_o, float* __restrict__ hn_o,
                                                          SeqParams sp) {
  extern __shared__ float4 seq_smem[];
  const int H = sp.H, B = sp.stride, S = H + 4, tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  float* sW = reinterpret_cast<float*>(seq_smem);  // [3 * kUPC][H]: row g * kUPC + u = W_hh[g * H + j0 + u][:]
  float* sh = sW + 3 * kUPC * H;                   // [32][H + 4]
  float* sred = sh + 32 * S;                       // [8][3 * kUPC][32]
  const int j0 = blockIdx.x * kUPC, H4 = H / 4, kslice = H / 8;
  for (int i = tid; i < 3 * kUPC * H4; i += 256) {
    const int row = i / H4, k4 = i % H4, g = row / kUPC, u = row % kUPC;
    reinterpret_cast<float4*>(sW)[i] = reinterpret_cast<const float4*>(whh + (size_t)(g * H + j0 + u) * H)[k4];
  }
  __syncthreads();
  // gate thread (b, u): biases once; W_ih x + b_ih of the NEXT step is fetched before the barrier it has to sit out
  const int gb = tid & 31, gu = tid >> 5, gj = j0 + gu;
  float bh0 = 0.f, bh1 = 0.f, bh2 = 0.f, gi0 = 0.f, gi1 = 0.f, gi2 = 0.f;
  if (tid < 32 * kUPC) { bh0 = bhh[gj]; bh1 = bhh[H + gj]; bh2 = bhh[2 * H + gj]; }
  auto fetch_gi = [&](int t) {
    if (tid < 32 * kUPC && t < sp.L && gb < seq_rows_alive(sp, t)) {
      const float* gir = gi + ((size_t)t * B + gb) * 3 * H;
      gi0 = gir[gj]; gi1 = gir[H + gj]; gi2 = gir[2 * H + gj];
    }
  };
  fetch_gi(0);
  // (the grid handle is taken once, before the loop: taken at the barrier, ptxas 12.9 spills 44 B in this kernel)
  cooperative_groups::grid_group grid = cooperative_groups::this_grid();
  for (int t = 0; t < sp.L; ++t) {
    const int nb = seq_rows_alive(sp, t);
    if (nb == 0) break;
    const size_t o = (size_t)t * B;
    for (int i = tid; i < nb * H4; i += 256) {  // h_{t-1}, written by every CTA in the previous step: read through L2
      const int b = i / H4, k4 = i % H4;
      *reinterpret_cast<float4*>(sh + b * S + 4 * k4) = __ldcg(reinterpret_cast<const float4*>(hs + (o + b) * H) + k4);
    }
    __syncthreads();
    float acc[3 * kUPC];
#pragma unroll
    for (int q = 0; q < 3 * kUPC; ++q) acc[q] = 0.f;
    if (lane < nb) {
      const float* hb = sh + lane * S + w * kslice;
      const float* wb = sW + w * kslice;
      for (int k = 0; k < kslice; k += 4) {
        const float4 hv = *reinterpret_cast<const float4*>(hb + k);
#pragma unroll
        for (int q = 0; q < 3 * kUPC; ++q) {
          const float4 wv = *reinterpret_cast<const float4*>(wb + q * H + k);
          acc[q] = fmaf(wv.x, hv.x, acc[q]); acc[q] = fmaf(wv.y, hv.y, acc[q]);
          acc[q] = fmaf(wv.z, hv.z, acc[q]); acc[q] = fmaf(wv.w, hv.w, acc[q]);
        }
      }
    }
#pragma unroll
    for (int q = 0; q < 3 * kUPC; ++q) sred[(w * 3 * kUPC + q) * 32 + lane] = acc[q];
    __syncthreads();
    if (tid < 32 * kUPC) {
      const int b = tid & 31, u = tid >> 5, j = j0 + u;
      if (b < nb) {
        float g3[3];
#pragma unroll
        for (int g = 0; g < 3; ++g) {
          float a = 0.f;
          for (int ww = 0; ww < 8; ++ww) a += sred[(ww * 3 * kUPC + g * kUPC + u) * 32 + b];
          g3[g] = a;
        }
        const float r = sigmoid_f32(gi0 + (g3[0] + bh0));
        const float z = sigmoid_f32(gi1 + (g3[1] + bh1));
        const float hn = g3[2] + bh2;
        const float n = tanhf(gi2 + r * hn);
        const float hp = sh[b * S + j];
        const size_t q = (o + b) * H + j;
        hs[q + (size_t)B * H] = (hp - n) * z + n;
        r_o[q] = r; z_o[q] = z; n_o[q] = n; hn_o[q] = hn;
      }
    }
    fetch_gi(t + 1);
    grid.sync();
  }
}

// Backward: for t = L-1..0, rows b < nb(t): dh = dout_t + carry; gate gradients -> dGi_t, dGh_t (as
// gru_bwd_step_kernel); carry = dh * z + dGh_t W_hh.  The CTA keeps the carry of its own 4 units on chip.
__global__ void __launch_bounds__(256) gru_seq_bwd_kernel(const float* __restrict__ whh, const float* __restrict__ dout,
                                                          const float* __restrict__ r_i, const float* __restrict__ z_i,
                                                          const float* __restrict__ n_i, const float* __restrict__ hn_i,
                                                          const float* __restrict__ hs, float* __restrict__ dgi,
                                                          float* dgh, float* __restrict__ carry_out, SeqParams sp) {
  extern __shared__ float4 seq_smem[];
  const int H = sp.H, B = sp.stride, H3 = 3 * H, CH = H3 / 4, S = CH + 4, rpw = CH / 8;
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5, j0 = blockIdx.x * kUPC;
  float4* sWT = seq_smem;                                 // [3H]: W_hh[row][j0 .. j0 + 3]
  float* sg = reinterpret_cast<float*>(sWT + H3);         // [2][32][CH + 4]
  float4* sred = reinterpret_cast<float4*>(sg + 2 * 32 * S);  // [8][32]
  float* scarry = reinterpret_cast<float*>(sred + 8 * 32);  // [32][4]
  for (int i = tid; i < H3; i += 256) sWT[i] = *reinterpret_cast<const float4*>(whh + (size_t)i * H + j0);
  if (tid < 32 * kUPC) scarry[tid] = 0.f;
  __syncthreads();
  // gate thread (b, u): the saved activations of the NEXT step are fetched while this step's product runs
  const int ab = tid >> 2, au = tid & 3, aj = j0 + au;
  float a_do = 0.f, a_r = 0.f, a_z = 0.f, a_n = 0.f, a_hn = 0.f, a_hp = 0.f;
  auto fetch_a = [&](int t) {
    if (tid < 32 * kUPC && t >= 0 && ab < seq_rows_alive(sp, t)) {
      const size_t q = ((size_t)t * B + ab) * H + aj;
      a_do = dout[q]; a_r = r_i[q]; a_z = z_i[q]; a_n = n_i[q]; a_hn = hn_i[q]; a_hp = hs[q];
    }
  };
  fetch_a(sp.L - 1);
  cooperative_groups::grid_group grid = cooperative_groups::this_grid();
  for (int t = sp.L - 1; t >= 0; --t) {  // lengths[0] == L: every step has at least one live row
    const int nb = seq_rows_alive(sp, t);
    const size_t o = (size_t)t * B;
    if (tid < 32 * kUPC && ab < nb) {
      const float dh = a_do + scarry[tid];
      const float r = a_r, z = a_z, n = a_n, hn = a_hn, hp = a_hp;
      const float dn = dh * (1.f - z), dz = dh * (hp - n);
      const float dan = dn * (1.f - n * n);
      const float dar = dan * hn * r * (1.f - r);
      const float daz = dz * z * (1.f - z);
      float* gi = dgi + (o + ab) * H3;
      float* gh = dgh + (o + ab) * H3;
      gi[aj] = dar; gi[H + aj] = daz; gi[2 * H + aj] = dan;
      gh[aj] = dar; gh[H + aj] = daz; gh[2 * H + aj] = dan * r;
      scarry[tid] = dh * z;
    }
    grid.sync();
    fetch_a(t - 1);
    // dGh_t (written by every CTA before the barrier) streams through two staging buffers: L2 -> smem copies
    // (cp.async.cg: L2 only, never a stale L1 line) of chunk c + 1 run under the product with chunk c
    auto stage = [&](int c) {
      float* dst = sg + (c & 1) * 32 * S;
      for (int i = tid; i < nb * (CH / 4); i += 256) {
        const int b = i / (CH / 4), c4 = i % (CH / 4);
        cp_async16(dst + b * S + 4 * c4, dgh + (o + b) * H3 + (size_t)c * CH + 4 * c4);
      }
      cp_async_commit();
    };
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    stage(0);
    for (int c = 0; c < 4; ++c) {
      if (c + 1 < 4) { stage(c + 1); cp_async_wait_but_one(); } else { cp_async_wait_all(); }
      __syncthreads();
      if (lane < nb) {
        const float* gb = sg + (c & 1) * 32 * S + lane * S + w * rpw;
        const float4* wt = sWT + c * CH + w * rpw;
        for (int rr = 0; rr < rpw; rr += 4) {
          const float4 g4 = *reinterpret_cast<const float4*>(gb + rr);
          const float4 w0 = wt[rr], w1 = wt[rr + 1], w2 = wt[rr + 2], w3 = wt[rr + 3];
          acc.x = fmaf(g4.x, w0.x, acc.x); acc.y = fmaf(g4.x, w0.y, acc.y); acc.z = fmaf(g4.x, w0.z, acc.z); acc.w = fmaf(g4.x, w0.w, acc.w);
          acc.x = fmaf(g4.y, w1.x, acc.x); acc.y = fmaf(g4.y, w1.y, acc.y); acc.z = fmaf(g4.y, w1.z, acc.z); acc.w = fmaf(g4.y, w1.w, acc.w);
          acc.x = fmaf(g4.z, w2.x, acc.x); acc.y = fmaf(g4.z, w2.y, acc.y); acc.z = fmaf(g4.z, w2.z, acc.z); acc.w = fmaf(g4.z, w2.w, acc.w);
          acc.x = fmaf(g4.w, w3.x, acc.x); acc.y = fmaf(g4.w, w3.y, acc.y); acc.z = fmaf(g4.w, w3.z, acc.z); acc.w = fmaf(g4.w, w3.w, acc.w);
        }
      }
      __syncthreads();  // the buffer of chunk c is free for chunk c + 2
    }
    sred[w * 32 + lane] = acc;
    __syncthreads();
    if (tid < 32 * kUPC && ab < nb) {
      float a = 0.f;
      for (int ww = 0; ww < 8; ++ww) a += reinterpret_cast<const float*>(sred + ww * 32 + ab)[au];
      scarry[tid] += a;
    }
    __syncthreads();
  }
  if (tid < 32 * kUPC) {
    const int b = tid >> 2, u = tid & 3;
    if (b < sp.B) carry_out[(size_t)b * H + j0 + u] = scarry[tid];
  }
}

// out[c][r] = in[r][c]
__global__ void transpose_kernel(const float* __restrict__ in, float* __restrict__ out, int R, int Cn) {
  __shared__ float tile[32][33];
  const int r0 = blockIdx.y * 32, c0 = blockIdx.x * 32;
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int r = r0 + i, c = c0 + threadIdx.x;
    if (r < R && c < Cn) tile[i][threadIdx.x] = in[(size_t)r * Cn + c];
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int c = c0 + i, r = r0 + threadIdx.x;
    if (r < R && c < Cn) out[(size_t)c * R + r] = tile[threadIdx.x][i];
  }
}

// GRU backward, elementwise part of one time step (b < nb):
//   dh = dout_t + carry ; gate gradients ; dGi_t, dGh_t ; carry <- dh * z   (the W_hh^T dGh term is a GEMM)
__global__ void gru_bwd_step_kernel(const float* __restrict__ dout_t, float* __restrict__ carry,
                                    const float* __restrict__ r_t, const float* __restrict__ z_t,
                                    const float* __restrict__ n_t, const float* __restrict__ hn_t,
                                    const float* __restrict__ hprev, float* __restrict__ dgi_t,
                                    float* __restrict__ dgh_t, int nb, int H) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= nb * H) return;
  const int b = q / H, j = q % H;
  const float dh = dout_t[q] + carry[q];
  const float r = r_t[q], z = z_t[q], n = n_t[q], hn = hn_t[q], hp = hprev[q];
  const float dn = dh * (1.f - z), dz = dh * (hp - n);
  const float dan = dn * (1.f - n * n);
  const float dar = dan * hn * r * (1.f - r);
  const float daz = dz * z * (1.f - z);
  float* gi = dgi_t + (size_t)b * 3 * H;
  float* gh = dgh_t + (size_t)b * 3 * H;
  gi[j] = dar; gi[H + j] = daz; gi[2 * H + j] = dan;
  gh[j] = dar; gh[H + j] = daz; gh[2 * H + j] = dan * r;
  carry[q] = dh * z;
}

// ---------------------------------------------------------------------------------------------
// Losses.  Thread (b, d) walks the time axis.
//   phase 1: running mean of the predictions, masked residual, per-dimension sums / counts
//   phase 2: gradient w.r.t. the per-step predictions (reverse running sum)
__global__ void loss_fwd_kernel(const float* __restrict__ mu, const float* __restrict__ x, float* __restrict__ diff,
                                float* __restrict__ sum_sq_d, float* __restrict__ cnt_d, float* __restrict__ nz_rows,
                                int L, int B, int D) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= B * D) return;
  const int b = q / D, d = q % D;
  float cum = 0.f, s = 0.f, c = 0.f, nz = 0.f;
  for (int t = 0; t + 1 < L; ++t) {
    const size_t o = ((size_t)t * B + b) * D + d;
    cum += mu[o];
    const float avg = cum * (1.0f / (float)(t + 1));          // cumsum * (1/steps), uisrnn.py:265-271
    const float truth = x[o + (size_t)B * D];                 // rnn_truth = rnn_input[1:]
    const float pred = (truth != 0.f) ? avg : 0.f;            // (rnn_truth != 0) * mean
    const float df = pred - truth;
    diff[o] = df;
    const float sq = df * df;
    s += sq;
    if (sq != 0.f) { c += 1.f; if (d == 0) nz += 1.f; }
  }
  atomicAdd(&sum_sq_d[d], s);
  atomicAdd(&cnt_d[d], c);
  if (d == 0) atomicAdd(nz_rows, nz);
}

__global__ void loss_bwd_kernel(const float* __restrict__ diff, const float* __restrict__ sigma2,
                                const float* __restrict__ nz_rows, float* __restrict__ dmu, int L, int B, int D) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= B * D) return;
  const int b = q / D, d = q % D;
  const float w = 1.f / (2.f * sigma2[d]);
  const float scale = 2.f * w / nz_rows[0];
  float acc = 0.f;
  dmu[((size_t)(L - 1) * B + b) * D + d] = 0.f;
  for (int t = L - 2; t >= 0; --t) {
    const size_t o = ((size_t)t * B + b) * D + d;
    acc += diff[o] * scale * (1.0f / (float)(t + 1));
    dmu[o] = acc;
  }
}

// scalars[0..2] = loss1, loss2, loss3 ; g_sigma2 written into the gradient buffer
__global__ void loss_scalar_kernel(const float* __restrict__ sum_sq_d, const float* __restrict__ cnt_d,
                                   const float* __restrict__ nz_rows, const float* __restrict__ sigma2,
                                   float sigma_alpha, float sigma_beta, float* __restrict__ g_sigma2,
                                   float* __restrict__ scalars, int D) {
  __shared__ float s1[256], s2[256];
  float l1 = 0.f, l2 = 0.f;
  const float nz = nz_rows[0];
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    const float sg = sigma2[d], nd = cnt_d[d];
    const float w = 1.f / (2.f * sg);
    l1 += sum_sq_d[d] * w;
    l2 += (2.f * sigma_alpha + nd + 2.f) / (2.f * nd) * logf(sg) + sigma_beta / (sg * nd);
    g_sigma2[d] = -(sum_sq_d[d] / nz) / (2.f * sg * sg) + ((2.f * sigma_alpha + nd + 2.f) / (2.f * nd)) / sg -
                  sigma_beta / (sg * sg * nd);
  }
  s1[threadIdx.x] = l1; s2[threadIdx.x] = l2;
  __syncthreads();
  for (int o = blockDim.x / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) { s1[threadIdx.x] += s1[threadIdx.x + o]; s2[threadIdx.x] += s2[threadIdx.x + o]; }
    __syncthreads();
  }
  if (threadIdx.x == 0) { scalars[0] = s1[0] / nz; scalars[1] = s2[0]; }
}

// ---------------------------------------------------------------------------------------------
// Optimiser.  Parameters live in one flat buffer; segment s covers [seg_off[s], seg_off[s+1]).
// grid (kSumsqBlocks, segments): partial[s][blockIdx.x]; then one block per segment folds the partials
constexpr int kSumsqBlocks = 64;
__global__ void seg_sumsq_partial_kernel(const float* __restrict__ v, const int* __restrict__ seg_off,
                                         float* __restrict__ partial) {
  __shared__ float sh[256];
  const int s = blockIdx.y;
  float a = 0.f;
  for (int i = seg_off[s] + blockIdx.x * 256 + threadIdx.x; i < seg_off[s + 1]; i += kSumsqBlocks * 256) a += v[i] * v[i];
  sh[threadIdx.x] = a;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) partial[s * kSumsqBlocks + blockIdx.x] = sh[0];
}
__global__ void seg_sumsq_final_kernel(const float* __restrict__ partial, float* __restrict__ out) {
  __shared__ float sh[kSumsqBlocks];
  const int s = blockIdx.x;
  sh[threadIdx.x] = partial[s * kSumsqBlocks + threadIdx.x];
  __syncthreads();
  for (int o = kSumsqBlocks / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) out[s] = sh[0];
}

// g += reg * p / ||p||  on the RNN segments (loss3 = reg * sum ||p||); scalars[2] = loss3
__global__ void reg_grad_kernel(const float* __restrict__ p, float* __restrict__ g, const int* __restrict__ seg_off,
                                const float* __restrict__ p_sumsq, float reg, int n_rnn_seg, float* __restrict__ scalars) {
  const int s = blockIdx.y;
  const float nrm = sqrtf(p_sumsq[s]);
  const int i = seg_off[s] + blockIdx.x * blockDim.x + threadIdx.x;
  if (i < seg_off[s + 1] && nrm > 0.f) g[i] += reg * p[i] / nrm;  // torch.norm'(0) = 0
  if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) {
    float l3 = 0.f;
    for (int q = 0; q < n_rnn_seg; ++q) l3 += sqrtf(p_sumsq[q]);
    scalars[2] = reg * l3;
  }
}

// clip (RNN segments only, torch.nn.utils.clip_grad_norm_) + Adam (torch.optim.Adam defaults) + clamp
__global__ void adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                            float* __restrict__ v, const float* __restrict__ g_sumsq, int n_rnn_seg, int rnn_end,
                            int sigma_begin, int total, float max_norm, float step_size, float bc2_sqrt,
                            int train_sigma2) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  if (i >= sigma_begin && !train_sigma2) return;
  float gi = g[i];
  if (i < rnn_end) {
    float tot = 0.f;
    for (int q = 0; q < n_rnn_seg; ++q) tot += g_sumsq[q];
    const float coef = fminf(max_norm / (sqrtf(tot) + 1e-6f), 1.0f);
    gi *= coef;
  }
  // 1 - beta is rounded from its exact value, as torch does with the Python doubles (1.f - 0.999f would be
  // 1.3e-5 relative off 0.001, and every update 6e-6 relative off torch's)
  const float b1 = 0.9f, b2 = 0.999f, one_m_b1 = 0.1f, one_m_b2 = 0.001f, eps = 1e-8f;
  const float mi = b1 * m[i] + one_m_b1 * gi;
  const float vi = b2 * v[i] + one_m_b2 * gi * gi;
  m[i] = mi; v[i] = vi;
  const float denom = sqrtf(vi) / bc2_sqrt + eps;
  float pi = p[i] - step_size * (mi / denom);
  if (i >= sigma_begin) pi = fmaxf(pi, 1e-6f);  // self.sigma2.data.clamp_(min=1e-6), uisrnn.py:295
  p[i] = pi;
}

// g[i] /= nz for i < n  (data-parallel path: gradients were accumulated without the 1/#rows factor)
__global__ void scale_by_inv_kernel(float* __restrict__ g, const float* __restrict__ nz, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) g[i] = g[i] / nz[0];
}

// Corpus path (fit() host data prep on the device, SURVEY 8(f) f1): a mini-batch is a gather of training rows.
// x[t][b][:] = 0 for t = 0 (the prepended zero frame, utils.py:243) and for t >= length_b (padding), else row
// index[begin_b + t - 1] converted to fp32.  The rows are either the trainer's own fp32 corpus (T = float,
// kTable = false: row r at rows + r * D) or the caller's rows read in place in their dtype (kTable = true: `rows` is
// a device table of row addresses, row r at ((const T* const*)rows)[r]).  Elements are loaded one by one, so a row
// needs only the alignment of T.
struct GatherCols { long long begin[32]; int length[32]; };
__device__ __forceinline__ float to_f32(float v) { return v; }
__device__ __forceinline__ float to_f32(double v) { return __double2float_rn(v); }  // = torch .float()
__device__ __forceinline__ float to_f32(__half v) { return __half2float(v); }       // exact
__device__ __forceinline__ float to_f32(__nv_bfloat16 v) { return __bfloat162float(v); }  // exact
// columns [b0, b0 + nbg) of a batch B columns wide; grid = L * nbg
template <typename T, bool kTable>
__global__ void gather_batch_kernel(const void* __restrict__ rows, const int* __restrict__ index, GatherCols cols,
                                    float* __restrict__ x, int nbg, int b0, int B, int D) {
  const int tt = blockIdx.x / nbg, bl = blockIdx.x % nbg;
  float* dst = x + ((size_t)tt * B + b0 + bl) * D;
  const bool live = tt >= 1 && tt < cols.length[bl];
  const T* src = nullptr;
  if (live) {
    const int r = index[cols.begin[bl] + tt - 1];
    src = kTable ? static_cast<const T* const*>(rows)[r] : static_cast<const T*>(rows) + (size_t)r * D;
  }
  for (int i = threadIdx.x; i < D; i += blockDim.x) dst[i] = live ? to_f32(src[i]) : 0.f;
}

// Inter-layer dropout of the stacked GRU in train mode (nn.GRU(dropout=p), uisrnn.py:39-41): element i of the output
// of layer `layer` in iteration `iter` is kept with probability 1 - p and scaled by 1 / (1 - p).  The keep decision
// is a pure function of (seed, iter, layer, i) -- a 32-bit integer hash, restated in tests/test_gpu_fit.py -- so the
// backward pass regenerates the mask instead of storing it.  (PyTorch draws its masks from the device generator /
// cuDNN dropout state; the streams differ, the distribution is the same.)
__host__ __device__ __forceinline__ unsigned dropout_hash(unsigned seed, unsigned iter, unsigned layer, unsigned i) {
  unsigned h = seed ^ (iter * 0x9E3779B1u) ^ (layer * 0x85EBCA77u) ^ (i * 0xC2B2AE3Du);
  h ^= h >> 16; h *= 0x7FEB352Du; h ^= h >> 15; h *= 0x846CA68Bu; h ^= h >> 16;
  return h;
}
// out[i] = in[i] * keep(i) / (1 - p); in == out is fine
__global__ void dropout_kernel(const float* __restrict__ in, float* __restrict__ out, size_t n, unsigned seed,
                               unsigned iter, unsigned layer, float p, float inv_keep) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    const float u = (float)(dropout_hash(seed, iter, layer, (unsigned)i) >> 8) * (1.0f / 16777216.0f);
    out[i] = u >= p ? in[i] * inv_keep : 0.f;
  }
}
__global__ void set_scalar_kernel(float* p, float v) { *p = v; }
// hs_l[b][:] = h0[l][:] for every batch column b and layer l (one launch instead of depth * B small copies)
__global__ void broadcast_h0_kernel(float* __restrict__ hs, const float* __restrict__ h0, size_t layer_stride, int B, int H) {
  const int l = blockIdx.y;
  for (int q = blockIdx.x * blockDim.x + threadIdx.x; q < B * H; q += gridDim.x * blockDim.x)
    hs[(size_t)l * layer_stride + q] = h0[(size_t)l * H + q % H];
}
__global__ void cast_rows_kernel(const double* __restrict__ in, float* __restrict__ out, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) out[i] = __double2float_rn(in[i]);  // = torch .float() of a float64 array
}

struct DBuf {
  float* p = nullptr;
  size_t cap = 0;
  int ensure(size_t n) {
    if (n <= cap) return 0;
    if (p) cudaFree(p);
    p = nullptr; cap = 0;
    cudaError_t e = cudaMalloc(&p, (n + n / 8 + 64) * sizeof(float));
    if (e != cudaSuccess) return api_fail(UIS_ERR_NOMEM, "cudaMalloc failed: %s", cudaGetErrorString(e));
    cap = n + n / 8 + 64;
    return 0;
  }
  void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
};

struct SplitCtx {
  float* partial = nullptr;     // [tiles][splits][64*64]
  size_t partial_cap = 0;       // floats
  unsigned* tile_tickets = nullptr;
  int ticket_cap = 0;
  float* colsum_partial = nullptr;  // [colsum_groups][kColsumSlices][32]
  unsigned* colsum_tickets = nullptr;
  int colsum_groups = 0;
};

// out[n] = sum_r A[r][n]; uses its own partial / ticket area behind the GEMMs' (sc.colsum_*)
inline void colsum(cudaStream_t st, const SplitCtx& sc, const float* A, float* out, int R, int N) {
  const int groups = (N + 31) / 32;
  int slices = (R >= 256 && groups <= sc.colsum_groups) ? kColsumSlices : 1;
  colsum_kernel<<<dim3(groups, slices), 256, 0, st>>>(A, out, R, N, sc.colsum_partial, sc.colsum_tickets);
}

template <bool TA, bool TB>
int gemm(cudaStream_t st, const SplitCtx& sc, const float* A, const float* B, const float* bias, const float* mask,
         float* C, int M, int N, int K, bool relu = false, bool acc = false) {
  if (M <= 0 || N <= 0) return 0;
  const bool big = M >= 128 && N >= 128;  // 128x128 tiles; tiny models keep the 64x64 kernel
  const int T = big ? 128 : 64;
  dim3 grid((N + T - 1) / T, (M + T - 1) / T, 1);
  const int tiles = grid.x * grid.y;
  int splits = 1;
  // fill the machine (>= 2 waves of CTAs) when the tile count is small and K is long
  const int want = big ? 296 : 592;
  while (splits < 16 && tiles * splits < want && K / (splits * 2) >= 128) splits *= 2;
  if (splits > 1 && ((size_t)tiles * splits * T * T > sc.partial_cap || tiles > sc.ticket_cap)) splits = 1;
  grid.z = splits;
  if (big)
    gemm128_kernel<TA, TB><<<grid, 256, 0, st>>>(A, B, bias, mask, C, M, N, K, relu ? 1 : 0, acc ? 1 : 0, sc.partial,
                                               sc.tile_tickets);
  else
    gemm_kernel<TA, TB><<<grid, 256, 0, st>>>(A, B, bias, mask, C, M, N, K, relu ? 1 : 0, acc ? 1 : 0, sc.partial,
                                            sc.tile_tickets);
  CUT(cudaGetLastError());
  return 0;
}

}  // namespace uis

constexpr int kMaxTrainDepth = 4;
constexpr int kMaxSegs = 4 * kMaxTrainDepth + 6;

struct uis_trainer {
  int device = 0, D = 0, H = 0, depth = 1;
  uis_train_hparams hp{};
  // parameter segments: [W_ih_l, W_hh_l, b_ih_l, b_hh_l] per layer, W1, b1, W2, b2, h0 [depth][H], sigma2
  int n_seg = 10, n_rnn_seg = 8;
  int seg_off_h[kMaxSegs + 1];
  int total = 0, rnn_end = 0, sigma_begin = 0;
  int seg_wih(int l) const { return 4 * l; }
  int seg_whh(int l) const { return 4 * l + 1; }
  int seg_bih(int l) const { return 4 * l + 2; }
  int seg_bhh(int l) const { return 4 * l + 3; }
  int seg_w1() const { return 4 * depth; }
  int seg_b1() const { return 4 * depth + 1; }
  int seg_w2() const { return 4 * depth + 2; }
  int seg_b2() const { return 4 * depth + 3; }
  int seg_h0() const { return 4 * depth + 4; }
  int seg_sigma2() const { return 4 * depth + 5; }
  long long step = 0, calls = 0;
  uis::DBuf params, grads, m, v, segbuf;  // segbuf: seg_off (as int bits) is separate below
  int* seg_off_d = nullptr;
  float* small = nullptr;  // [sum_sq_d D][cnt_d D][nz 1][scalars 4][p_sumsq 32][g_sumsq 32]
  // gi, hs, r, z, n, hn: one slab per layer (the backward pass needs every layer's activations); xin: the (dropped)
  // input sequence of layers >= 1
  uis::DBuf x, gi, hs, r, z, n, hn, xin, a1, mu, diff, dmu, dz1, dout, dgi, dgh, carry, whh_t, ghbuf, partial, skpart;
  unsigned* tickets = nullptr;
  uis::SplitCtx sc;
  uis::DBuf gemm_partial, loss_hist;
  unsigned* gemm_tickets = nullptr;
  long long hist_cap = 0;
  // pinned staging for the batch (two buffers in flight) so that steps are truly asynchronous
  float* pin[2] = {nullptr, nullptr};
  size_t pin_cap = 0;
  cudaEvent_t pin_ev[2] = {nullptr, nullptr};
  int pin_idx = 0;
  int seq_mode = -1;  // -1 unknown, 0 per-step launches, 1 persistent cooperative kernels
  // corpus path: training rows (fp32) + flat gather indices + per-sub-sequence offsets (host copy).  After
  // uis_trainer_set_corpus_device the rows are the caller's, read in place through the device table row_addr
  // (corpus is then empty).
  uis::DBuf corpus;
  const void* const* row_addr = nullptr;
  int row_dtype = UIS_DTYPE_F32;
  cudaEvent_t legacy_done = nullptr;  // set_corpus_device: the caller's stream waits for the legacy-stream work
  int* corpus_index = nullptr;
  long long corpus_rows = 0;
  std::vector<long long> sub_off;
};

namespace {

// Tail of an iteration: regulariser gradient + loss3, then (mode 0) clip + Adam + clamp; records the losses.
int finish_step(uis_trainer* t, cudaStream_t st, int mode, float* losses_out) {
  using namespace uis;
  const int D = t->D;
  float* P = t->params.p;
  float* G = t->grads.p;
  const int* so = t->seg_off_h;
  float* nz = t->small + 2 * D;
  float* scalars = nz + 1; float* p_sumsq = scalars + 4; float* g_sumsq = p_sumsq + 32;
  const int nrs = t->n_rnn_seg;  // the tensors of rnn_model.parameters(): regularised one by one, clipped as a group
  seg_sumsq_partial_kernel<<<dim3(kSumsqBlocks, nrs), 256, 0, st>>>(P, t->seg_off_d, t->partial.p);
  seg_sumsq_final_kernel<<<nrs, kSumsqBlocks, 0, st>>>(t->partial.p, p_sumsq);
  {
    int maxseg = 0;
    for (int s = 0; s < nrs; ++s) maxseg = std::max(maxseg, so[s + 1] - so[s]);
    dim3 grid((maxseg + 255) / 256, nrs);
    reg_grad_kernel<<<grid, 256, 0, st>>>(P, G, t->seg_off_d, p_sumsq, t->hp.regularization_weight, nrs, scalars);
  }
  CUT(cudaGetLastError());
  if (mode == 0) {
    seg_sumsq_partial_kernel<<<dim3(kSumsqBlocks, nrs), 256, 0, st>>>(G, t->seg_off_d, t->partial.p);
    seg_sumsq_final_kernel<<<nrs, kSumsqBlocks, 0, st>>>(t->partial.p, g_sumsq);
    t->step += 1;
    // torch.optim.Adam (defaults): step_size = lr / (1 - beta1^t) and sqrt(1 - beta2^t) are Python doubles
    const double bc1 = 1.0 - std::pow(0.9, (double)t->step), bc2 = 1.0 - std::pow(0.999, (double)t->step);
    adam_kernel<<<(t->total + 255) / 256, 256, 0, st>>>(P, G, t->m.p, t->v.p, g_sumsq, nrs, t->rnn_end, t->sigma_begin,
                                                        t->total, t->hp.grad_max_norm,
                                                        (float)((double)t->hp.learning_rate / bc1),
                                                        (float)std::sqrt(bc2), t->hp.train_sigma2);
    CUT(cudaGetLastError());
  }
  // loss history on the device: slot (calls mod capacity); losses_out == NULL => fully asynchronous step
  if (!t->loss_hist.p) {
    if (int rc = t->loss_hist.ensure(3 * 4096)) return rc;
    t->hist_cap = 4096;
  }
  CUT(cudaMemcpyAsync(t->loss_hist.p + 3 * (t->calls % t->hist_cap), scalars, 3 * sizeof(float), cudaMemcpyDeviceToDevice, st));
  t->calls += 1;
  if (losses_out) {
    CUT(cudaMemcpyAsync(losses_out, scalars, 3 * sizeof(float), cudaMemcpyDeviceToHost, st));
    CUT(cudaStreamSynchronize(st));
  }
  return 0;
}

}  // namespace

extern "C" {

int uis_trainer_create(uis_trainer** out, int device, int D, int H, const float* const* params /*[4 * depth + 6] host*/,
                       const uis_train_hparams* hp) {
  if (!out || !params || !hp) return uis::api_fail(UIS_ERR_INVALID, "null argument");
  *out = nullptr;
  if (D < 1 || H < 1 || H > 4096 || D > 4096) return uis::api_fail(UIS_ERR_INVALID, "bad shape");
  const int depth = hp->rnn_depth <= 0 ? 1 : hp->rnn_depth;
  if (depth > kMaxTrainDepth)
    return uis::api_fail(UIS_ERR_UNSUPPORTED, "rnn_depth=%d: the training kernels take 1..%d stacked GRU layers", depth, kMaxTrainDepth);
  if (!(hp->rnn_dropout >= 0.f && hp->rnn_dropout < 1.f)) return uis::api_fail(UIS_ERR_INVALID, "rnn_dropout must be in [0, 1)");
  uis::DeviceGuard device_guard_(device);
  CUT(device_guard_.status);
  uis_trainer* t = new uis_trainer();
  t->device = device; t->D = D; t->H = H; t->hp = *hp; t->depth = depth;
  t->n_seg = 4 * depth + 6; t->n_rnn_seg = 4 * depth + 4;
  int sizes[kMaxSegs];
  for (int l = 0; l < depth; ++l) {
    sizes[t->seg_wih(l)] = 3 * H * (l == 0 ? D : H);
    sizes[t->seg_whh(l)] = 3 * H * H;
    sizes[t->seg_bih(l)] = 3 * H;
    sizes[t->seg_bhh(l)] = 3 * H;
  }
  sizes[t->seg_w1()] = H * H; sizes[t->seg_b1()] = H; sizes[t->seg_w2()] = D * H; sizes[t->seg_b2()] = D;
  sizes[t->seg_h0()] = depth * H; sizes[t->seg_sigma2()] = D;
  t->seg_off_h[0] = 0;
  for (int s = 0; s < t->n_seg; ++s) t->seg_off_h[s + 1] = t->seg_off_h[s] + sizes[s];
  t->total = t->seg_off_h[t->n_seg];
  t->rnn_end = t->seg_off_h[t->seg_h0()];
  t->sigma_begin = t->seg_off_h[t->seg_sigma2()];
  auto body = [&]() -> int {
    if (int rc = t->params.ensure(t->total)) return rc;
    if (int rc = t->grads.ensure(t->total)) return rc;
    if (int rc = t->m.ensure(t->total)) return rc;
    if (int rc = t->v.ensure(t->total)) return rc;
    for (int s = 0; s < t->n_seg; ++s) {
      if (!params[s]) return uis::api_fail(UIS_ERR_INVALID, "NULL parameter %d", s);
      CUT(cudaMemcpy(t->params.p + t->seg_off_h[s], params[s], (size_t)sizes[s] * 4, cudaMemcpyDefault));
    }
    CUT(cudaMemset(t->m.p, 0, (size_t)t->total * 4));
    CUT(cudaMemset(t->v.p, 0, (size_t)t->total * 4));
    CUT(cudaMalloc(&t->seg_off_d, sizeof(t->seg_off_h)));
    CUT(cudaMemcpy(t->seg_off_d, t->seg_off_h, sizeof(t->seg_off_h), cudaMemcpyHostToDevice));
    CUT(cudaMalloc(&t->small, (size_t)(2 * D + 128) * 4));
    // finish_step's per-segment sum-of-squares partials: allocated here, not by the first iteration, because a
    // data-parallel rank that holds no batch column calls uis_trainer_comm_apply before it has ever stepped
    if (int rc = t->partial.ensure((size_t)32 * uis::kSumsqBlocks)) return rc;
    CUT(cudaMalloc(&t->tickets, 256 * sizeof(unsigned)));
    CUT(cudaMemset(t->tickets, 0, 256 * sizeof(unsigned)));
    CUT(cudaMalloc(&t->gemm_tickets, 4096 * sizeof(unsigned)));
    CUT(cudaMemset(t->gemm_tickets, 0, 4096 * sizeof(unsigned)));
    if (int rc = t->gemm_partial.ensure((size_t)4096 * 4096)) return rc;  // 64 MB of split-K partial tiles
    t->sc.partial = t->gemm_partial.p; t->sc.partial_cap = t->gemm_partial.cap; t->sc.tile_tickets = t->gemm_tickets; t->sc.ticket_cap = 4096;
    t->sc.colsum_groups = (std::max(3 * H, D) + 31) / 32;
    CUT(cudaMalloc(&t->sc.colsum_partial, (size_t)t->sc.colsum_groups * uis::kColsumSlices * 32 * sizeof(float)));
    CUT(cudaMalloc(&t->sc.colsum_tickets, (size_t)t->sc.colsum_groups * sizeof(unsigned)));
    CUT(cudaMemset(t->sc.colsum_tickets, 0, (size_t)t->sc.colsum_groups * sizeof(unsigned)));
    return 0;
  };
  if (int rc = body()) { uis_trainer_destroy(t); return rc; }
  *out = t;
  return 0;
}

int uis_trainer_destroy(uis_trainer* t) {
  if (!t) return 0;
  uis::DeviceGuard device_guard_(t->device);
  uis::DBuf* bufs[] = {&t->params, &t->grads, &t->m, &t->v, &t->segbuf, &t->x, &t->gi, &t->hs, &t->r, &t->z, &t->n,
                       &t->hn, &t->xin, &t->a1, &t->mu, &t->diff, &t->dmu, &t->dz1, &t->dout, &t->dgi, &t->dgh, &t->carry, &t->whh_t, &t->ghbuf,
                       &t->partial, &t->skpart, &t->gemm_partial, &t->loss_hist};
  for (auto* b : bufs) b->release();
  if (t->seg_off_d) cudaFree(t->seg_off_d);
  if (t->small) cudaFree(t->small);
  if (t->tickets) cudaFree(t->tickets);
  if (t->gemm_tickets) cudaFree(t->gemm_tickets);
  if (t->sc.colsum_partial) cudaFree(t->sc.colsum_partial);
  if (t->sc.colsum_tickets) cudaFree(t->sc.colsum_tickets);
  if (t->corpus_index) cudaFree(t->corpus_index);
  t->corpus.release();
  if (t->legacy_done) cudaEventDestroy(t->legacy_done);
  for (int i = 0; i < 2; ++i) {
    if (t->pin[i]) cudaFreeHost(t->pin[i]);
    if (t->pin_ev[i]) cudaEventDestroy(t->pin_ev[i]);
  }
  delete t;
  return 0;
}

namespace {
size_t seq_fwd_smem(int H) { return (size_t)(3 * uis::kUPC * H + 32 * (H + 4) + 8 * 3 * uis::kUPC * 32) * 4; }
size_t seq_bwd_smem(int H) { return (size_t)3 * H * 16 + (size_t)2 * 32 * (3 * H / 4 + 4) * 4 + 8 * 32 * 16 + 32 * uis::kUPC * 4; }

// Decides once per trainer whether the persistent recurrence kernels can run (H % 128 == 0, the H / 4 CTAs
// co-resident, cooperative launch supported); UISRNN_B200_TRAIN_STEPWISE=1 forces the per-step launches.
int seq_setup(uis_trainer* t) {
  t->seq_mode = 0;
  const char* env = std::getenv("UISRNN_B200_TRAIN_STEPWISE");
  if (env && env[0] == '1') return 0;
  const int H = t->H;
  if (H % 128 != 0) return 0;
  int coop = 0, sms = 0, max_smem = 0;
  CUT(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, t->device));
  CUT(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, t->device));
  CUT(cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, t->device));
  if (!coop || seq_fwd_smem(H) > (size_t)max_smem || seq_bwd_smem(H) > (size_t)max_smem) return 0;
  CUT(cudaFuncSetAttribute(uis::gru_seq_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)seq_fwd_smem(H)));
  CUT(cudaFuncSetAttribute(uis::gru_seq_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)seq_bwd_smem(H)));
  int occ_f = 0, occ_b = 0;
  CUT(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_f, uis::gru_seq_fwd_kernel, 256, seq_fwd_smem(H)));
  CUT(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_b, uis::gru_seq_bwd_kernel, 256, seq_bwd_smem(H)));
  if (occ_f * sms < H / uis::kUPC || occ_b * sms < H / uis::kUPC) return 0;
  t->seq_mode = 1;
  return 0;
}

int check_lengths(const int32_t* lengths, int B, int L) {
  if (B < 1 || B > (1 << 20)) return uis::api_fail(UIS_ERR_INVALID, "batch width %d", B);
  if (L < 2) return uis::api_fail(UIS_ERR_INVALID, "L < 2");
  for (int b = 0; b < B; ++b) {
    if (lengths[b] < 1 || lengths[b] > L || (b > 0 && lengths[b] > lengths[b - 1]) || (b == 0 && lengths[0] != L))
      return uis::api_fail(UIS_ERR_INVALID, "lengths must be sorted descending with lengths[0] == L");
  }
  return 0;
}
int run_iteration(uis_trainer* t, const int32_t* lengths, int B, int L, int mode, float* losses_out, cudaStream_t st,
                  const float* x_host, const long long* col_begin);
}  // namespace

// One iteration on a host batch.  x_host: fp32 [L][B][D] zero-padded (row 0 = zero frame), lengths[B] sorted
// descending (each includes the zero frame).
int uis_trainer_step(uis_trainer* t, const float* x_host, const int32_t* lengths, int B, int L, int mode,
                     float* losses_out /*[3] host*/, void* stream) {
  if (!t || !x_host || !lengths) return uis::api_fail(UIS_ERR_INVALID, "null argument");
  if (int rc = check_lengths(lengths, B, L)) return rc;
  uis::DeviceGuard device_guard_(t->device);
  CUT(device_guard_.status);
  return run_iteration(t, lengths, B, L, mode, losses_out, static_cast<cudaStream_t>(stream), x_host, nullptr);
}

// Training set on the device: rows [n_rows][D] float64 host (cast to fp32 on the device, as the reference's
// torch.from_numpy(...).float() does per batch, utils.py:245), index = the concatenated row indices of every
// sub-sequence of utils.resize_sequence, offsets[n_sub + 1] its prefix sums.
namespace {
// The host-side checks both set_corpus entry points make of the gather plan.
int check_corpus(int64_t n_rows, const int32_t* index, int64_t n_index, const int64_t* offsets, int32_t n_sub) {
  if (n_rows < 1 || n_sub < 1 || n_index < 0 || offsets[0] != 0 || offsets[n_sub] != n_index)
    return uis::api_fail(UIS_ERR_INVALID, "inconsistent corpus sizes");
  for (int64_t i = 0; i < n_index; ++i)
    if (index[i] < 0 || index[i] >= n_rows) return uis::api_fail(UIS_ERR_INVALID, "corpus index out of range");
  for (int32_t k = 0; k < n_sub; ++k)
    if (offsets[k + 1] < offsets[k]) return uis::api_fail(UIS_ERR_INVALID, "corpus offsets must be non-decreasing");
  return 0;
}
}  // namespace

int uis_trainer_set_corpus(uis_trainer* t, const double* rows, int64_t n_rows, const int32_t* index, int64_t n_index,
                           const int64_t* offsets, int32_t n_sub) {
  if (!t || !rows || !index || !offsets) return uis::api_fail(UIS_ERR_INVALID, "null argument");
  if (int rc = check_corpus(n_rows, index, n_index, offsets, n_sub)) return rc;
  uis::DeviceGuard device_guard_(t->device);
  CUT(device_guard_.status);
  const size_t n = (size_t)n_rows * t->D;
  if (int rc = t->corpus.ensure(n)) return rc;
  double* tmp = nullptr;
  const size_t chunk_rows = std::min<size_t>((size_t)n_rows, (size_t)1 << 16);
  CUT(cudaMalloc(&tmp, chunk_rows * t->D * sizeof(double)));
  for (size_t r0 = 0; r0 < (size_t)n_rows; r0 += chunk_rows) {
    const size_t nr = std::min(chunk_rows, (size_t)n_rows - r0), ne = nr * t->D;
    cudaError_t e = cudaMemcpy(tmp, rows + r0 * t->D, ne * sizeof(double), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) {
      uis::cast_rows_kernel<<<1024, 256>>>(tmp, t->corpus.p + r0 * t->D, ne);
      e = cudaDeviceSynchronize();
    }
    if (e != cudaSuccess) { cudaFree(tmp); return uis::api_fail(UIS_ERR_CUDA, "corpus upload: %s", cudaGetErrorString(e)); }
  }
  cudaFree(tmp);
  if (t->corpus_index) { cudaFree(t->corpus_index); t->corpus_index = nullptr; }
  CUT(cudaMalloc(&t->corpus_index, std::max<size_t>(1, (size_t)n_index) * sizeof(int)));
  CUT(cudaMemcpy(t->corpus_index, index, (size_t)n_index * sizeof(int), cudaMemcpyHostToDevice));
  t->corpus_rows = n_rows;
  t->row_addr = nullptr;
  t->sub_off.assign(offsets, offsets + n_sub + 1);
  return 0;
}

// Training set left where the caller holds it: row r is D elements of `dtype` at the device address row_addr[r]
// (row_addr: a device table of n_rows addresses), read in place by every later uis_trainer_step_corpus.  index and
// offsets as in uis_trainer_set_corpus.  uis_trainer_create initialises the trainer on the legacy default stream and
// the index goes up there too; `stream` (which may be a non-blocking stream) waits for that work on an event, so
// neither the host nor the legacy stream waits for earlier work on `stream`.
int uis_trainer_set_corpus_device(uis_trainer* t, const void* const* row_addr, int32_t dtype, int64_t n_rows,
                                  const int32_t* index, int64_t n_index, const int64_t* offsets, int32_t n_sub,
                                  void* stream) {
  if (!row_addr || !index || !offsets) return uis::api_fail(UIS_ERR_INVALID, "null argument");
  if (dtype < UIS_DTYPE_F32 || dtype > UIS_DTYPE_F64) return uis::api_fail(UIS_ERR_INVALID, "unknown dtype %d", dtype);
  if (int rc = check_corpus(n_rows, index, n_index, offsets, n_sub)) return rc;
  if (!t) return uis::api_fail(UIS_ERR_INVALID, "trainer is NULL");
  uis::DeviceGuard device_guard_(t->device);
  CUT(device_guard_.status);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  t->corpus.release();  // (cudaFree waits for the steps that may still read an earlier corpus)
  if (t->corpus_index) { cudaFree(t->corpus_index); t->corpus_index = nullptr; }
  CUT(cudaMalloc(&t->corpus_index, std::max<size_t>(1, (size_t)n_index) * sizeof(int)));
  CUT(cudaMemcpyAsync(t->corpus_index, index, (size_t)n_index * sizeof(int), cudaMemcpyHostToDevice, cudaStreamLegacy));
  if (!t->legacy_done) CUT(cudaEventCreateWithFlags(&t->legacy_done, cudaEventDisableTiming));
  CUT(cudaEventRecord(t->legacy_done, cudaStreamLegacy));
  CUT(cudaStreamWaitEvent(st, t->legacy_done, 0));
  t->row_addr = row_addr;
  t->row_dtype = dtype;
  t->corpus_rows = n_rows;
  t->sub_off.assign(offsets, offsets + n_sub + 1);
  return 0;
}

// One iteration on the batch whose columns are sub-sequences chosen[0..B) of the corpus (lengths + 1 sorted
// descending, as utils.pack_sequence orders them).  Nothing but `chosen` crosses the bus.
int uis_trainer_step_corpus(uis_trainer* t, const int32_t* chosen, int B, int mode, float* losses_out, void* stream) {
  if (!t || !chosen) return uis::api_fail(UIS_ERR_INVALID, "null argument");
  if (t->sub_off.empty()) return uis::api_fail(UIS_ERR_INVALID, "uis_trainer_set_corpus has not been called");
  if (B < 1 || B > (1 << 20)) return uis::api_fail(UIS_ERR_INVALID, "batch width %d", B);
  std::vector<long long> begin(B);
  std::vector<int32_t> lengths(B);
  const long long n_sub = (long long)t->sub_off.size() - 1;
  for (int b = 0; b < B; ++b) {
    if (chosen[b] < 0 || chosen[b] >= n_sub) return uis::api_fail(UIS_ERR_INVALID, "sub-sequence id out of range");
    begin[b] = t->sub_off[chosen[b]];
    lengths[b] = (int32_t)(t->sub_off[chosen[b] + 1] - t->sub_off[chosen[b]]) + 1;  // + the zero frame
  }
  if (int rc = check_lengths(lengths.data(), B, lengths[0])) return rc;
  uis::DeviceGuard device_guard_(t->device);
  CUT(device_guard_.status);
  return run_iteration(t, lengths.data(), B, lengths[0], mode, losses_out, static_cast<cudaStream_t>(stream), nullptr, begin.data());
}

}  // extern "C"

namespace {
// One iteration.  The batch comes either from the host (x_host: fp32 [L][B][D] zero-padded, row 0 = zero frame)
// or from the device-resident corpus (cols).  lengths[B] sorted descending (each includes the zero frame).
// mode 0: full step (forward, backward, clip, Adam); mode 1: forward + backward only (gradients can be read
// back with uis_trainer_get, for tests); mode 2: data-parallel shard.
int run_iteration(uis_trainer* t, const int32_t* lengths, int B, int L, int mode, float* losses_out, cudaStream_t st,
                  const float* x_host, const long long* col_begin) {
  using namespace uis;
  const int D = t->D, H = t->H, depth = t->depth;
  const size_t R = (size_t)L * B;
  const size_t RH = R * H, RB = (R + B) * H;  // per-layer slab sizes (hs has one extra time step: h_{-1})
  if (int rc = t->x.ensure(R * D)) return rc;
  if (int rc = t->gi.ensure((size_t)depth * R * 3 * H)) return rc;
  if (int rc = t->hs.ensure((size_t)depth * RB)) return rc;
  if (int rc = t->r.ensure((size_t)depth * RH)) return rc;
  if (int rc = t->z.ensure((size_t)depth * RH)) return rc;
  if (int rc = t->n.ensure((size_t)depth * RH)) return rc;
  if (int rc = t->hn.ensure((size_t)depth * RH)) return rc;
  const bool drop = depth > 1 && t->hp.rnn_dropout > 0.f;
  if (drop)
    if (int rc = t->xin.ensure((size_t)(depth - 1) * RH)) return rc;
  if (int rc = t->a1.ensure(RH)) return rc;
  if (int rc = t->mu.ensure(R * D)) return rc;
  if (int rc = t->diff.ensure(R * D)) return rc;
  if (int rc = t->dmu.ensure(R * D)) return rc;
  if (int rc = t->dz1.ensure(RH)) return rc;
  if (int rc = t->dout.ensure(RH)) return rc;
  if (int rc = t->dgi.ensure(R * 3 * H)) return rc;
  if (int rc = t->dgh.ensure(R * 3 * H)) return rc;
  if (int rc = t->carry.ensure((size_t)B * H)) return rc;
  if (int rc = t->whh_t.ensure((size_t)3 * H * H)) return rc;
  if (int rc = t->ghbuf.ensure((size_t)32 * 3 * H)) return rc;
  if (int rc = t->skpart.ensure((size_t)((3 * H + 63) / 64) * kSplit * 32 * 64)) return rc;
  if ((3 * H + 63) / 64 > 256) return api_fail(UIS_ERR_UNSUPPORTED, "hidden size too large for the training kernels");
  if (R * 3 * H > (size_t)0x7fffffff) return api_fail(UIS_ERR_UNSUPPORTED, "batch of %d x %d rows is too large", L, B);
  float* P = t->params.p;
  float* G = t->grads.p;
  const int* so = t->seg_off_h;
  float* sum_sq_d = t->small; float* cnt_d = t->small + D; float* nz = t->small + 2 * D;
  float* scalars = nz + 1;
  // batch columns are processed by the recurrence in groups of <= 32 (one warp lane per column)
  const int n_groups = (B + 31) / 32;
  auto group_rows = [&](int g, int tt) {  // live columns of group g at time tt (lengths are sorted descending)
    const int b0 = 32 * g, nbg = std::min(32, B - b0);
    int c = 0;
    while (c < nbg && lengths[b0 + c] > tt) ++c;
    return c;
  };

  if (col_begin) {
    for (int g = 0; g < n_groups; ++g) {
      const int b0 = 32 * g, nbg = std::min(32, B - b0);
      GatherCols cols{};
      for (int b = 0; b < nbg; ++b) { cols.begin[b] = col_begin[b0 + b]; cols.length[b] = lengths[b0 + b]; }
      const dim3 grid((unsigned)(L * nbg));
      const void* rows = t->row_addr;
      if (!t->row_addr)
        gather_batch_kernel<float, false><<<grid, 128, 0, st>>>(t->corpus.p, t->corpus_index, cols, t->x.p, nbg, b0, B, D);
      else if (t->row_dtype == UIS_DTYPE_F32)
        gather_batch_kernel<float, true><<<grid, 128, 0, st>>>(rows, t->corpus_index, cols, t->x.p, nbg, b0, B, D);
      else if (t->row_dtype == UIS_DTYPE_F16)
        gather_batch_kernel<__half, true><<<grid, 128, 0, st>>>(rows, t->corpus_index, cols, t->x.p, nbg, b0, B, D);
      else if (t->row_dtype == UIS_DTYPE_BF16)
        gather_batch_kernel<__nv_bfloat16, true><<<grid, 128, 0, st>>>(rows, t->corpus_index, cols, t->x.p, nbg, b0, B, D);
      else
        gather_batch_kernel<double, true><<<grid, 128, 0, st>>>(rows, t->corpus_index, cols, t->x.p, nbg, b0, B, D);
    }
    CUT(cudaGetLastError());
  } else {  // stage the batch in pinned memory: the H2D copy then overlaps the previous iteration's kernels
    const size_t bytes = R * D * 4;
    if (bytes > t->pin_cap) {
      for (int i = 0; i < 2; ++i) {
        if (t->pin_ev[i]) CUT(cudaEventSynchronize(t->pin_ev[i]));
        if (t->pin[i]) cudaFreeHost(t->pin[i]);
        t->pin[i] = nullptr;
        CUT(cudaMallocHost(&t->pin[i], bytes + bytes / 4));
        if (!t->pin_ev[i]) CUT(cudaEventCreateWithFlags(&t->pin_ev[i], cudaEventDisableTiming));
      }
      t->pin_cap = bytes + bytes / 4;
    }
    const int pi = t->pin_idx;
    t->pin_idx ^= 1;
    CUT(cudaEventSynchronize(t->pin_ev[pi]));  // the copy that last used this buffer has finished
    std::memcpy(t->pin[pi], x_host, bytes);
    CUT(cudaMemcpyAsync(t->x.p, t->pin[pi], bytes, cudaMemcpyHostToDevice, st));
    CUT(cudaEventRecord(t->pin_ev[pi], st));
  }
  CUT(cudaMemsetAsync(t->hs.p, 0, (size_t)depth * RB * 4, st));
  CUT(cudaMemsetAsync(t->small, 0, (size_t)(2 * D + 128) * 4, st));
  CUT(cudaMemsetAsync(G, 0, (size_t)t->total * 4, st));
  CUT(cudaMemsetAsync(t->dgi.p, 0, R * 3 * H * 4, st));
  CUT(cudaMemsetAsync(t->dgh.p, 0, R * 3 * H * 4, st));
  // h_{-1} of layer l = rnn_init_hidden[l] repeated over the batch (uisrnn.py:262)
  broadcast_h0_kernel<<<dim3((unsigned)std::min<size_t>(((size_t)B * H + 255) / 256, 256), depth), 256, 0, st>>>(
      t->hs.p, P + so[t->seg_h0()], RB, B, H);
  CUT(cudaGetLastError());
  if (t->seq_mode < 0) {
    if (int rc = seq_setup(t)) return rc;
  }
  const unsigned it_no = (unsigned)t->calls;  // dropout masks: a function of (seed, iteration, layer, element)
  const unsigned seed = (unsigned)(t->hp.dropout_seed ^ (t->hp.dropout_seed >> 32));
  const float keep_inv = drop ? 1.0f / (1.0f - t->hp.rnn_dropout) : 1.0f;
  const int drop_blocks = (int)std::min<size_t>((RH + 255) / 256, 132 * 8);
  // input sequence of layer l: the batch itself, or the (dropped) output sequence of the layer below
  auto layer_in = [&](int l) -> const float* {
    if (l == 0) return t->x.p;
    return drop ? t->xin.p + (size_t)(l - 1) * RH : t->hs.p + (size_t)(l - 1) * RB + (size_t)B * H;
  };

  // ---- forward
  for (int l = 0; l < depth; ++l) {
    float* gi_l = t->gi.p + (size_t)l * R * 3 * H;
    float* hs_l = t->hs.p + (size_t)l * RB;
    float* r_l = t->r.p + (size_t)l * RH; float* z_l = t->z.p + (size_t)l * RH;
    float* n_l = t->n.p + (size_t)l * RH; float* hn_l = t->hn.p + (size_t)l * RH;
    const float* whh = P + so[t->seg_whh(l)];
    const float* bhh = P + so[t->seg_bhh(l)];
    if (int rc = gemm<false, true>(st, t->sc, layer_in(l), P + so[t->seg_wih(l)], P + so[t->seg_bih(l)], nullptr, gi_l, (int)R,
                                   3 * H, l == 0 ? D : H)) return rc;
    if (t->seq_mode == 0) {  // k-major copy of W_hh for the per-step recurrent products (the weights change every iteration)
      dim3 tg((H + 31) / 32, (3 * H + 31) / 32), tb(32, 8);
      transpose_kernel<<<tg, tb, 0, st>>>(whh, t->whh_t.p, 3 * H, H);
    }
    for (int g = 0; g < n_groups; ++g) {
      const int b0 = 32 * g, nbg = std::min(32, B - b0), Lg = lengths[b0];
      if (t->seq_mode == 1) {
        SeqParams sp{};
        for (int b = 0; b < 32; ++b) sp.length[b] = b < nbg ? lengths[b0 + b] : 0;
        sp.L = Lg; sp.B = nbg; sp.H = H; sp.stride = B;
        const float* a_whh = whh; const float* a_bhh = bhh; const float* a_gi = gi_l + (size_t)b0 * 3 * H;
        float* a_hs = hs_l + (size_t)b0 * H; float* a_r = r_l + (size_t)b0 * H; float* a_z = z_l + (size_t)b0 * H;
        float* a_n = n_l + (size_t)b0 * H; float* a_hn = hn_l + (size_t)b0 * H;
        void* args[] = {&a_whh, &a_bhh, &a_gi, &a_hs, &a_r, &a_z, &a_n, &a_hn, &sp};
        CUT(cudaLaunchCooperativeKernel((const void*)gru_seq_fwd_kernel, dim3(H / kUPC), dim3(256), args, seq_fwd_smem(H), st));
      } else {
        for (int tt = 0; tt < Lg; ++tt) {
          const int nb = group_rows(g, tt);
          if (nb == 0) break;
          const size_t o = (size_t)tt * B + b0;
          splitk_gemm_kernel<<<dim3((3 * H + 63) / 64, kSplit), 256, 0, st>>>(hs_l + o * H, H, t->whh_t.p, t->ghbuf.p, 3 * H,
                                                                              nb, 3 * H, H, 0, t->skpart.p, t->tickets);
          gru_gate_fwd_kernel<<<(nb * H + 255) / 256, 256, 0, st>>>(t->ghbuf.p, bhh, gi_l + o * 3 * H, hs_l + o * H,
                                                                    hs_l + (o + B) * H, r_l + o * H, z_l + o * H,
                                                                    n_l + o * H, hn_l + o * H, nb, H);
        }
      }
    }
    CUT(cudaGetLastError());
    if (drop && l + 1 < depth) {
      dropout_kernel<<<drop_blocks, 256, 0, st>>>(hs_l + (size_t)B * H, t->xin.p + (size_t)l * RH, RH, seed, it_no, (unsigned)l,
                                                 t->hp.rnn_dropout, keep_inv);
      CUT(cudaGetLastError());
    }
  }
  const float* out = t->hs.p + (size_t)(depth - 1) * RB + (size_t)B * H;  // out[t] = h_t of the top layer; padded rows stay zero
  if (int rc = gemm<false, true>(st, t->sc, out, P + so[t->seg_w1()], P + so[t->seg_b1()], nullptr, t->a1.p, (int)R, H, H, true)) return rc;
  if (int rc = gemm<false, true>(st, t->sc, t->a1.p, P + so[t->seg_w2()], P + so[t->seg_b2()], nullptr, t->mu.p, (int)R, D, H)) return rc;
  const int bd_blocks = (B * D + 255) / 256;
  loss_fwd_kernel<<<bd_blocks, 256, 0, st>>>(t->mu.p, t->x.p, t->diff.p, sum_sq_d, cnt_d, nz, L, B, D);
  // mode 2 (data-parallel shard): the row count is global, so gradients are accumulated WITHOUT the 1/nz
  // factor (they are linear in it) and normalised after the all-reduce, in uis_trainer_comm_apply()
  const float* nz_for_bwd = nz;
  if (mode == 2) {
    set_scalar_kernel<<<1, 1, 0, st>>>(scalars + 3, 1.0f);  // (a pageable H2D copy would synchronise the stream)
    nz_for_bwd = scalars + 3;
  } else {
    loss_scalar_kernel<<<1, 256, 0, st>>>(sum_sq_d, cnt_d, nz, P + so[t->seg_sigma2()], t->hp.sigma_alpha, t->hp.sigma_beta,
                                         G + so[t->seg_sigma2()], scalars, D);
  }
  // ---- backward
  loss_bwd_kernel<<<bd_blocks, 256, 0, st>>>(t->diff.p, P + so[t->seg_sigma2()], nz_for_bwd, t->dmu.p, L, B, D);
  CUT(cudaGetLastError());
  if (int rc = gemm<true, false>(st, t->sc, t->dmu.p, t->a1.p, nullptr, nullptr, G + so[t->seg_w2()], D, H, (int)R)) return rc;
  colsum(st, t->sc, t->dmu.p, G + so[t->seg_b2()], (int)R, D);
  if (int rc = gemm<false, false>(st, t->sc, t->dmu.p, P + so[t->seg_w2()], nullptr, t->a1.p, t->dz1.p, (int)R, H, D)) return rc;  // * relu'
  if (int rc = gemm<true, false>(st, t->sc, t->dz1.p, out, nullptr, nullptr, G + so[t->seg_w1()], H, H, (int)R)) return rc;
  colsum(st, t->sc, t->dz1.p, G + so[t->seg_b1()], (int)R, H);
  if (int rc = gemm<false, false>(st, t->sc, t->dz1.p, P + so[t->seg_w1()], nullptr, nullptr, t->dout.p, (int)R, H, H)) return rc;
  for (int l = depth - 1; l >= 0; --l) {  // dout = gradient w.r.t. the output sequence of layer l
    const float* hs_l = t->hs.p + (size_t)l * RB;
    const float* r_l = t->r.p + (size_t)l * RH; const float* z_l = t->z.p + (size_t)l * RH;
    const float* n_l = t->n.p + (size_t)l * RH; const float* hn_l = t->hn.p + (size_t)l * RH;
    const float* whh = P + so[t->seg_whh(l)];
    CUT(cudaMemsetAsync(t->carry.p, 0, (size_t)B * H * 4, st));
    for (int g = 0; g < n_groups; ++g) {
      const int b0 = 32 * g, nbg = std::min(32, B - b0), Lg = lengths[b0];
      if (t->seq_mode == 1) {
        SeqParams sp{};
        for (int b = 0; b < 32; ++b) sp.length[b] = b < nbg ? lengths[b0 + b] : 0;
        sp.L = Lg; sp.B = nbg; sp.H = H; sp.stride = B;
        const float* a_whh = whh; const float* a_dout = t->dout.p + (size_t)b0 * H; const float* a_r = r_l + (size_t)b0 * H;
        const float* a_z = z_l + (size_t)b0 * H; const float* a_n = n_l + (size_t)b0 * H; const float* a_hn = hn_l + (size_t)b0 * H;
        const float* a_hs = hs_l + (size_t)b0 * H;
        float* a_dgi = t->dgi.p + (size_t)b0 * 3 * H; float* a_dgh = t->dgh.p + (size_t)b0 * 3 * H;
        float* a_carry = t->carry.p + (size_t)b0 * H;
        void* args[] = {&a_whh, &a_dout, &a_r, &a_z, &a_n, &a_hn, &a_hs, &a_dgi, &a_dgh, &a_carry, &sp};
        CUT(cudaLaunchCooperativeKernel((const void*)gru_seq_bwd_kernel, dim3(H / kUPC), dim3(256), args, seq_bwd_smem(H), st));
      } else {
        for (int tt = Lg - 1; tt >= 0; --tt) {
          const int nb = group_rows(g, tt);
          if (nb == 0) continue;
          const size_t o = (size_t)tt * B + b0;
          gru_bwd_step_kernel<<<(nb * H + 255) / 256, 256, 0, st>>>(t->dout.p + o * H, t->carry.p + (size_t)b0 * H, r_l + o * H,
                                                                    z_l + o * H, n_l + o * H, hn_l + o * H, hs_l + o * H,
                                                                    t->dgi.p + o * 3 * H, t->dgh.p + o * 3 * H, nb, H);
          // carry[b] += dGh_t[b] * W_hh   (W_hh stored [3H][H] = [K][N])
          splitk_gemm_kernel<<<dim3((H + 63) / 64, kSplit), 256, 0, st>>>(t->dgh.p + o * 3 * H, 3 * H, whh,
                                                                          t->carry.p + (size_t)b0 * H, H, nb, H, 3 * H, 1,
                                                                          t->skpart.p, t->tickets);
        }
      }
    }
    CUT(cudaGetLastError());
    if (int rc = gemm<true, false>(st, t->sc, t->dgi.p, layer_in(l), nullptr, nullptr, G + so[t->seg_wih(l)], 3 * H,
                                   l == 0 ? D : H, (int)R)) return rc;
    if (int rc = gemm<true, false>(st, t->sc, t->dgh.p, hs_l, nullptr, nullptr, G + so[t->seg_whh(l)], 3 * H, H, (int)R)) return rc;
    colsum(st, t->sc, t->dgi.p, G + so[t->seg_bih(l)], (int)R, 3 * H);
    colsum(st, t->sc, t->dgh.p, G + so[t->seg_bhh(l)], (int)R, 3 * H);
    colsum(st, t->sc, t->carry.p, G + so[t->seg_h0()] + (size_t)l * H, B, H);  // d h0 = sum_b d h_{-1}
    if (l > 0) {  // gradient w.r.t. this layer's input sequence = (through the dropout mask) the output of layer l - 1
      if (int rc = gemm<false, false>(st, t->sc, t->dgi.p, P + so[t->seg_wih(l)], nullptr, nullptr, t->dout.p, (int)R, H, 3 * H)) return rc;
      if (drop) {
        dropout_kernel<<<drop_blocks, 256, 0, st>>>(t->dout.p, t->dout.p, RH, seed, it_no, (unsigned)(l - 1), t->hp.rnn_dropout, keep_inv);
        CUT(cudaGetLastError());
      }
    }
  }
  if (mode == 2) return 0;  // gradients + statistics stay on the device for uis_trainer_comm_export()
  return finish_step(t, st, mode, losses_out);
}
}  // namespace

extern "C" {

// Losses of the last `count` (<= 4096) calls to uis_trainer_step, oldest first: out[count][3] (host).  Synchronises.
int uis_trainer_losses(uis_trainer* t, int count, float* out) {
  if (!t || !out || count < 0) return uis::api_fail(UIS_ERR_INVALID, "bad argument");
  if (count > t->calls || count > t->hist_cap) return uis::api_fail(UIS_ERR_INVALID, "only %lld steps recorded", t->calls);
  uis::DeviceGuard device_guard_(t->device);
  CUT(device_guard_.status);
  CUT(cudaDeviceSynchronize());
  for (int i = 0; i < count; ++i) {
    const long long slot = (t->calls - count + i) % t->hist_cap;
    CUT(cudaMemcpy(out + 3 * i, t->loss_hist.p + 3 * slot, 3 * sizeof(float), cudaMemcpyDeviceToHost));
  }
  return 0;
}

// ---- data-parallel fit(): one all-reduce(sum) per iteration over [unnormalised gradients of the RNN
// parameters and h0 | per-dimension residual sums | per-dimension counts | row count] (SURVEY 8(e)).
int64_t uis_trainer_comm_size(uis_trainer* t) { return t ? (int64_t)t->sigma_begin + 2 * t->D + 1 : 0; }

int uis_trainer_comm_export(uis_trainer* t, float* dev_buf, void* stream) {
  if (!t || !dev_buf) return uis::api_fail(UIS_ERR_INVALID, "null argument");
  uis::DeviceGuard device_guard_(t->device);
  CUT(device_guard_.status);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  CUT(cudaMemcpyAsync(dev_buf, t->grads.p, (size_t)t->sigma_begin * 4, cudaMemcpyDeviceToDevice, st));
  CUT(cudaMemcpyAsync(dev_buf + t->sigma_begin, t->small, (size_t)(2 * t->D + 1) * 4, cudaMemcpyDeviceToDevice, st));
  return 0;
}

int uis_trainer_comm_apply(uis_trainer* t, const float* dev_buf, void* stream) {
  if (!t || !dev_buf) return uis::api_fail(UIS_ERR_INVALID, "null argument");
  uis::DeviceGuard device_guard_(t->device);
  CUT(device_guard_.status);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int D = t->D;
  CUT(cudaMemcpyAsync(t->grads.p, dev_buf, (size_t)t->sigma_begin * 4, cudaMemcpyDeviceToDevice, st));
  CUT(cudaMemcpyAsync(t->small, dev_buf + t->sigma_begin, (size_t)(2 * D + 1) * 4, cudaMemcpyDeviceToDevice, st));
  float* nz = t->small + 2 * D;
  uis::scale_by_inv_kernel<<<(t->sigma_begin + 255) / 256, 256, 0, st>>>(t->grads.p, nz, t->sigma_begin);
  uis::loss_scalar_kernel<<<1, 256, 0, st>>>(t->small, t->small + D, nz, t->params.p + t->seg_off_h[t->seg_sigma2()],
                                            t->hp.sigma_alpha, t->hp.sigma_beta, t->grads.p + t->seg_off_h[t->seg_sigma2()],
                                            nz + 1, D);
  CUT(cudaGetLastError());
  return finish_step(t, st, 0, nullptr);
}

// what: 0 = parameters, 1 = gradients of the last step.  out[4 * depth + 6] host buffers (any may be NULL).
int uis_trainer_get(uis_trainer* t, int what, float* const* out) {
  if (!t || !out) return uis::api_fail(UIS_ERR_INVALID, "null argument");
  uis::DeviceGuard device_guard_(t->device);
  CUT(device_guard_.status);
  CUT(cudaDeviceSynchronize());
  const float* src = what == 0 ? t->params.p : t->grads.p;
  for (int s = 0; s < t->n_seg; ++s)
    if (out[s])
      CUT(cudaMemcpy(out[s], src + t->seg_off_h[s], (size_t)(t->seg_off_h[s + 1] - t->seg_off_h[s]) * 4,
                     cudaMemcpyDeviceToHost));
  return 0;
}

}  // extern "C"
