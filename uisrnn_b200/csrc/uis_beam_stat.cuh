// Stationary-weights (latency) mode of the beam kernel: ONE utterance is advanced by a group of kStatGroup = 32 CTAs that
// keep the whole weight set resident in shared memory for the lifetime of the kernel.
//
// Why: with one utterance in flight a beam step is a chain of three small matrix products (uisrnn.py:45-52) whose cost
// in the streaming kernels is the time to pull 4.7 MB of weights through a TMA ring every step -- bound by the latency
// of the L2 -> shared-memory round trip (96 KB in flight per CTA), also in the cluster mode.  4.7 MB do not fit one thread-block cluster (16 x 227 KB), but they
// fit 32 CTAs: CTA q owns the rows of 16 hidden units of W_hh (48 rows), 16 rows of W1 and 8 rows of W2 (72 x 512 fp32
// = 147 KB) and never loads them again.  Row split, so no partial sums travel: every CTA computes its rows of the
// product for all columns, writes them where the next product reads them -- the new slots of the (group-shared) slot
// pool for h' and the running mean, a small L2 scratch for a = relu(W1 h' + b1) -- and the group meets at a barrier in
// global memory (cooperative launch: the CTAs are co-resident).  Three barriers per beam step.  The selection phases
// run replicated in every CTA of the group (as in the cluster mode) on the shared pool; reads of data another CTA
// produced bypass L1 (ld.global.cg).
#pragma once
#include "uis_common.cuh"

namespace uis {

constexpr int kStatGroup = 32;  // CTAs per utterance

template <int H, int D>
struct StatCfg {
  static constexpr int GS = kStatGroup;
  static constexpr int UG = H / GS;           // hidden units (and W1 rows) per CTA
  static constexpr int R0 = 3 * UG;           // GRU rows per CTA (gate-major: r block, z block, n block)
  static constexpr int R1 = H / GS;           // W1 rows per CTA
  static constexpr int R2 = D / GS;           // W2 rows per CTA
  static constexpr int ROWS = R0 + R1 + R2;
  static constexpr int LD = H + 1;            // padded row stride (floats): conflict-free column access
  static constexpr unsigned BYTES = (unsigned)ROWS * LD * 4;
  static_assert(H % GS == 0 && D % GS == 0, "row split over the group");
};

// Barrier of the CTAs of one group through a counter in global memory.  Every consumer thread calls it; `epoch` counts
// the barriers passed (identical in all CTAs).  (A variant with one release-store flag per CTA watched by the 32 lanes
// of a warp was measured slower: 29.8 us per beam step against 24.9.)  Bounded spin: a lost CTA traps (a CUDA error in
// uis_get_stats) instead of hanging the device.
template <int NT>
__device__ __forceinline__ void stat_group_sync(unsigned* bar, unsigned& epoch, int tid) {
  named_bar_sync(1, NT);  // every thread's global writes of this phase are ordered before thread 0's fence
  epoch += 1;
  if (tid == 0) {
    __threadfence();
    atomicAdd(bar, 1u);
    const unsigned target = epoch * (unsigned)kStatGroup;
    unsigned v = 0;
    const long long t0 = clock64();
    unsigned spins = 0;
    for (;;) {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(bar) : "memory");
      if (v >= target) break;
      if ((++spins & 0x3ffu) == 0 && clock64() - t0 > 8000000000ll) __trap();
    }
    __threadfence();
  }
  named_bar_sync(1, NT);
}

// Resident weight rows of CTA `q` of the group: sW[row_local][k], row stride LD.
//   rows [0, R0):       W_hh rows g * H + q * UG + u  (row_local = g * UG + u)
//   rows [R0, R0+R1):   W1 rows q * R1 + u
//   rows [R0+R1, ROWS): W2 rows q * R2 + u
// The global arrays are the k-major transposes (whh_t [H][3H], w1_t [H][H], w2_t [H][D]).
template <int H, int D, int NT>
__device__ __forceinline__ void stat_load_weights(float* sW, const float* whh_t, const float* w1_t, const float* w2_t, int q,
                                                  int tid) {
  using S = StatCfg<H, D>;
  for (int i = tid; i < S::R0 * H; i += NT) {
    const int k = i / S::R0, r = i % S::R0, g = r / S::UG, u = r % S::UG;
    sW[(size_t)r * S::LD + k] = whh_t[(size_t)k * 3 * H + g * H + q * S::UG + u];
  }
  for (int i = tid; i < S::R1 * H; i += NT) {
    const int k = i / S::R1, r = i % S::R1;
    sW[(size_t)(S::R0 + r) * S::LD + k] = w1_t[(size_t)k * H + q * S::R1 + r];
  }
  for (int i = tid; i < S::R2 * H; i += NT) {
    const int k = i / S::R2, r = i % S::R2;
    sW[(size_t)(S::R0 + S::R1 + r) * S::LD + k] = w2_t[(size_t)k * D + q * S::R2 + r];
  }
}

// P[s][r][0 .. 4 * NC) = sum over k = s, s + KS, ... of sW[row0 + r][k] * X[k][0 .. 4 * NC)   (KS = NT / NR k-phases, fixed
// order; NC = float4 column groups actually in use, so that a typical step with <= 8 columns does 2/3 of the work)
template <int H, int NR, int CP, int NT, int NC>
__device__ __forceinline__ void stat_dot_nc(const float* sW, int ld, int row0, const float* X, float* P, int tid) {
  constexpr int KS = NT / NR;
  static_assert(CP % 4 == 0 && KS >= 1 && 4 * NC <= CP, "columns in float4 groups");
  const int r = tid % NR, s = tid / NR;
  if (s < KS) {
    float acc[4 * NC];
#pragma unroll
    for (int m = 0; m < 4 * NC; ++m) acc[m] = 0.f;
    const float* w = sW + (size_t)(row0 + r) * ld;
#pragma unroll 4
    for (int k = s; k < H; k += KS) {
      const float wk = w[k];
      const float4* x4 = reinterpret_cast<const float4*>(X + (size_t)k * CP);
#pragma unroll
      for (int c = 0; c < NC; ++c) {
        const float4 v = x4[c];
        acc[4 * c + 0] = fmaf(wk, v.x, acc[4 * c + 0]);
        acc[4 * c + 1] = fmaf(wk, v.y, acc[4 * c + 1]);
        acc[4 * c + 2] = fmaf(wk, v.z, acc[4 * c + 2]);
        acc[4 * c + 3] = fmaf(wk, v.w, acc[4 * c + 3]);
      }
    }
    float4* dst = reinterpret_cast<float4*>(P + ((size_t)s * NR + r) * CP);
#pragma unroll
    for (int c = 0; c < NC; ++c) dst[c] = make_float4(acc[4 * c], acc[4 * c + 1], acc[4 * c + 2], acc[4 * c + 3]);
  }
}
template <int H, int NR, int CP, int NT>
__device__ __forceinline__ void stat_dot(const float* sW, int ld, int row0, const float* X, float* P, int Mp, int tid) {
  static_assert(CP == 12, "column groups 1..3");
  if (Mp <= 4) stat_dot_nc<H, NR, CP, NT, 1>(sW, ld, row0, X, P, tid);
  else if (Mp <= 8) stat_dot_nc<H, NR, CP, NT, 2>(sW, ld, row0, X, P, tid);
  else stat_dot_nc<H, NR, CP, NT, 3>(sW, ld, row0, X, P, tid);
}
template <int NR, int CP, int NT>
__device__ __forceinline__ float stat_sum(const float* P, int r, int m) {
  constexpr int KS = NT / NR;
  float v = 0.f;
#pragma unroll
  for (int s = 0; s < KS; ++s) v = __fadd_rn(v, P[((size_t)s * NR + r) * CP + m]);
  return v;
}

}  // namespace uis
