// Tensor-core weight pass of the beam kernel (warpgroup MMA / tensor-map TMA, sm_90a).
//
// Same arithmetic as run_pass() in uis_beam.cuh -- h' = GRU(x_t, h_src), a = relu(W1 h' + b1), m = W2 a + b2 of the
// reference's CoreRNN.forward for the step's distinct source states -- but the three matrix products run on the
// tensor cores (wgmma) at fp32-grade accuracy:
//
//   * every weight w is split once, at uis_model_create, into two fp16 planes  w * 2^s = hi + lo  (22 significant
//     bits; s = a per-matrix power of two) stored K-major [2 * ROWS][H]; the planes are the A operand, streamed through
//     a shared-memory ring by tensor-map TMA (cp.async.bulk.tensor.2d, 128-byte swizzle, boxes of 128 rows x 64 k =
//     16 KB); each of the two consumer warpgroups multiplies the 64 rows of a box that are its own (m64 instructions);
//   * the hidden columns of the pass are split the same way by the consumer warps and stay in shared memory as the
//     B operand: per 64-wide k atom, rows [0, N) hold the hi halves and rows [N, 2N) the lo halves * 2^11 of the N
//     columns, so ONE instruction with N' = 2N multiplies a weight box with both:  D[:, 0:N] += A * Bhi,
//     D[:, N:2N] += A * Blo * 2^11 (the fold scales it back; the lo halves stay normal fp16 numbers, with all 11 bits,
//     when a loose bound on the columns leaves their values far below 2^14);
//   * per 128-row tile the lo boxes go first, then the hi boxes: the tensor core adds into its fp32 accumulator
//     with truncation, and the small products cost nothing while the accumulator is still small (max |error| 2.7e-6
//     against fp64 for 512-term sums of magnitude ~3; the fp32 FMA chain of the FFMA kernel: 2.3e-6);
//   * accumulators live in registers (m64 x 2N fp32 = N registers per thread); a warpgroup keeps one box of MMAs in
//     flight behind the one it issues and returns a ring box to the TMA producer as soon as its MMAs have completed.
//
// The cost of an m64 x N' x 16 MMA hardly depends on N' <= 96, so the kernel runs up to 6 utterances (lanes) per CTA and
// gives all their columns to one pass.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include "uis_common.cuh"

namespace uis {

constexpr int kTcBoxBytes = 16384;  // 128 rows x 64 k, fp16
constexpr int kTcColumns = 48;      // columns per pass: the one instantiated N

template <int H, int D, int N>
struct TcCfg {
  static constexpr int KA = H / 64;                       // 64-wide k atoms
  static constexpr int UT = H / 128;                      // hidden-unit tiles
  static constexpr int T1 = 3 * UT, T2 = H / 128, T3 = D / 128;  // 128-row tiles of W_hh, W1, W2
  static constexpr int TILES = T1 + T2 + T3;
  static constexpr int ROWS = 3 * H + H + D;              // rows of one plane
  static constexpr int NP = 2 * N;                        // B rows / accumulator columns per tile
  static constexpr int NACC = NP / 2;                     // accumulator registers per thread (m64 x NP over 128 threads)
  static constexpr int NV = N / 2;                        // folded (hi + lo) values per thread and tile
  static constexpr int ATOM_BYTES = NP * 128;             // one k atom of the B operand
  static constexpr int BOP_BYTES = KA * ATOM_BYTES;
  static constexpr int STAGES = 4;                        // ring depth (boxes)
  static_assert(H % 128 == 0 && D % 128 == 0, "tensor-core pass: 128-row tiles");
  static_assert(NP == 96, "wgmma instantiation: N = 48 columns");
};

// ---- PTX wrappers ---------------------------------------------------------------------------------------------
// shared-memory matrix descriptor, K-major, 128-byte swizzle: rows of 128 B, 8-row groups 1024 B apart
__device__ __forceinline__ uint64_t tc_desc_sw128(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3fff);  // start address, 16-byte units
  d |= (uint64_t)1 << 16;                  // leading byte offset (unused for swizzled K-major)
  d |= (uint64_t)(1024 >> 4) << 32;        // stride byte offset between 8-row groups
  d |= (uint64_t)1 << 62;                  // SWIZZLE_128B
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int PENDING>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(PENDING) : "memory"); }

// D (m64 x NP, fp32, registers) (+)= A (m64 x k16, fp16, shared) * B (k16 x NP, fp16, shared); both operands K-major.
// Accumulator register 4 i + 2 h + e of lane l in warp w of the warpgroup: row 16 w + l / 4 + 8 h, column 8 i + 2 (l % 4) + e.
template <int NP> struct Wgmma;
template <> struct Wgmma<96> {
  static __device__ __forceinline__ void mma(float (&d)[48], uint64_t adesc, uint64_t bdesc, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %50, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n96k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, %48, %49, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
        : "l"(adesc), "l"(bdesc), "r"(acc)
        : "memory");
  }
};

__device__ __forceinline__ void tc_tma_load_2d(void* dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}

// Bounded wait of the tensor-core pipeline: a protocol error must trap -- and surface as a CUDA error in
// uis_get_stats -- instead of hanging the device (~4 s at 2 GHz).
__device__ __forceinline__ void tc_mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  unsigned spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++spins & 0x3ffu) == 0 && clock64() - t0 > 8000000000ll) __trap();
  }
}

// Wait for an mbarrier phase, giving up when the consumer warps have announced the end of the kernel.
__device__ __forceinline__ bool tc_wait_or_done(uint64_t* bar, uint32_t parity, volatile int* done_flag) {
  for (;;) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity), "r"(4000u)  // park for at most ~4 us, then look at the flag
        : "memory");
    if (ok) return true;
    if (*done_flag) return false;
  }
}

// elect.sync: true in exactly one (the same) lane of a converged warp
__device__ __forceinline__ bool tc_elect_one() {
  uint32_t pred;
  asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
  return pred != 0;
}

struct TcBars {
  uint64_t* full;    // [STAGES]   TMA -> consumer warpgroups
  uint64_t* empty;   // [STAGES]   consumer warps -> TMA
};

// 128-row tile t of the pass -> first row inside one plane (W_hh tiles ordered (unit tile, gate): the three gate
// tiles of a unit tile are consecutive, so the GRU epilogue of unit tile u can run after 3 tiles)
template <class TC, int H>
__device__ __forceinline__ int tc_tile_row0(int t) {
  if (t < TC::T1) return (t % 3) * H + (t / 3) * 128;
  return 3 * H + (t - TC::T1) * 128;  // W1 rows, then W2 rows (contiguous after W_hh)
}

// ---- TMA producer (one warp, one elected lane issues): the box sequence of a pass is the same for every pass, so it
// free-runs ahead of the MMAs by the depth of the ring
template <class TC, int H>
__device__ void tc_producer_loop(const CUtensorMap* wmap, unsigned char* ring, const TcBars& b, volatile int* done_flag) {
  unsigned it = 0;
  bool run = true;
  while (run) {
    for (int t = 0; t < TC::TILES && run; ++t) {
      const int row0 = tc_tile_row0<TC, H>(t);
      for (int pl = 0; pl < 2 && run; ++pl) {  // plane 0 = lo, 1 = hi
        for (int ka = 0; ka < TC::KA; ++ka, ++it) {
          const unsigned s = it % TC::STAGES, ph = (it / TC::STAGES) & 1;
          if (!tc_wait_or_done(&b.empty[s], ph ^ 1, done_flag)) { run = false; break; }
          if (tc_elect_one()) {
            mbar_arrive_expect_tx(&b.full[s], kTcBoxBytes);
            tc_tma_load_2d(ring + (size_t)s * kTcBoxBytes, wmap, ka * 64, pl * TC::ROWS + row0, &b.full[s]);
          }
          __syncwarp();
        }
      }
    }
  }
  // boxes that were prefetched for a pass that never came: wait until they have landed before the CTA exits
  for (unsigned j = (it > (unsigned)TC::STAGES) ? it - TC::STAGES : 0; j < it; ++j)
    tc_mbar_wait(&b.full[j % TC::STAGES], (j / TC::STAGES) & 1);
}

// ---- one 128-row tile (consumer warpgroup `wg`: rows 64 wg .. 64 wg + 63 of it) ----------------------------------
// 2 * KA ring boxes -- the lo plane, then the hi plane -- times 4 k-steps of 16 inside each 64-wide swizzle atom
// (+32 bytes = +2 descriptor units each).  `box` counts the ring boxes consumed so far (identical in every consumer
// thread).  tstat (thread 0 only, else null): [0] cycles waiting for a box to land, [1] cycles waiting for MMAs.
template <class TC>
__device__ __forceinline__ void tc_tile(float (&acc)[TC::NACC], const unsigned char* ring, const unsigned char* bop,
                                        const TcBars& b, unsigned& box, int wg, int lane, long long* tstat) {
  const uint64_t desc0 = tc_desc_sw128(0);  // every field but the start address
  const uint32_t a16 = (smem_u32(ring) + (uint32_t)wg * (kTcBoxBytes / 2)) >> 4, b16 = smem_u32(bop) >> 4;
#pragma unroll
  for (int i = 0; i < TC::NACC; ++i) acc[i] = 0.f;
  unsigned prev = 0;
#pragma unroll 1
  for (int q = 0; q < 2 * TC::KA; ++q, ++box) {
    const unsigned s = box % TC::STAGES, par = (box / TC::STAGES) & 1u;
    if (!mbar_try_wait(&b.full[s], par)) {
      const long long w0 = tstat ? clock64() : 0;
      tc_mbar_wait(&b.full[s], par);
      if (tstat) tstat[0] += clock64() - w0;
    }
    const uint64_t adesc = desc0 + (uint64_t)(a16 + s * (kTcBoxBytes >> 4));
    const uint64_t bdesc = desc0 + (uint64_t)(b16 + (uint32_t)(q % TC::KA) * (TC::ATOM_BYTES >> 4));
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) Wgmma<TC::NP>::mma(acc, adesc + 2 * kk, bdesc + 2 * kk, (q | kk) != 0);
    wgmma_commit();
    if (q > 0) {  // the previous box's MMAs have completed: its ring stage goes back to the producer
      wgmma_wait<1>();
      __syncwarp();
      if (lane == 0) mbar_arrive(&b.empty[prev]);
    }
    prev = s;
  }
  const long long w0 = tstat ? clock64() : 0;
  wgmma_wait<0>();
  if (tstat) tstat[1] += clock64() - w0;
  __syncwarp();
  if (lane == 0) mbar_arrive(&b.empty[prev]);
}

// hi + lo column halves of a finished tile, scaled back: v[4 i + 2 h + e] <- row 8 h, column 8 i + 2 (lane % 4) + e.
// The lo columns hold lo * 2^11 (tc_gather_b): the FMA scales them back exactly and rounds once.
template <class TC>
__device__ __forceinline__ void tc_fold(const float (&acc)[TC::NACC], float (&v)[TC::NV], float inv) {
  constexpr int LO = TC::NACC / 2;  // register offset of the lo halves (columns N .. 2N - 1)
#pragma unroll
  for (int i = 0; i < TC::NV; ++i) v[i] = __fmul_rn(__fmaf_rn(acc[LO + i], 0x1p-11f, acc[i]), inv);
}

// ---- consumer warps: B operand ---------------------------------------------------------------------------------
// bop[(ka, row, 128 B)]: element (n, k) of plane pl -> atom k / 64, row pl * N + n, 16-byte chunk
// ((k % 64) / 8) ^ (row % 8), byte (k % 8) * 2   (the canonical K-major SWIZZLE_128B layout; N % 8 == 0)
template <int H, int N, int NTHREADS, class SrcFn>
__device__ __forceinline__ void tc_gather_b(unsigned char* bop, SrcFn src, int Mp, float scale, int tid) {
  constexpr int PPC = H / 2;            // float2 pairs per column
  constexpr int CG = NTHREADS / PPC;    // columns handled side by side
  static_assert(NTHREADS % PPC == 0 && CG >= 1, "gather mapping");
  const int pair = tid % PPC, cg = tid / PPC;
  const int k = 2 * pair;
  const uint32_t koff = (uint32_t)(k >> 6) * (2u * N * 128u) + (uint32_t)(k & 7) * 2u;
  const uint32_t kchunk = (uint32_t)(k & 63) >> 3;
  constexpr int UNR = 8;
  for (int m0 = cg; m0 < Mp; m0 += CG * UNR) {
    float2 v[UNR];
#pragma unroll
    for (int u = 0; u < UNR; ++u) {
      const int m = m0 + u * CG;
      v[u] = (m < Mp) ? *reinterpret_cast<const float2*>(src(m) + k) : make_float2(0.f, 0.f);
    }
#pragma unroll
    for (int u = 0; u < UNR; ++u) {
      const int m = m0 + u * CG;
      if (m < Mp) {
        const float x0 = v[u].x * scale, x1 = v[u].y * scale;
        const __half h0 = __float2half_rn(x0), h1 = __float2half_rn(x1);
        // lo * 2^11 (exact before the rounding; |lo * 2^11| <= |hi|): stays a normal fp16 number, with its 11 bits,
        // down to |x| ~ 2^-14 where x's own scale (a loose bound on the column) left the unscaled lo subnormal
        const __half l0 = __float2half_rn((x0 - __half2float(h0)) * 2048.f);
        const __half l1 = __float2half_rn((x1 - __half2float(h1)) * 2048.f);
        const uint32_t off = koff + (uint32_t)m * 128u + ((kchunk ^ ((uint32_t)m & 7u)) << 4);
        *reinterpret_cast<__half2*>(bop + off) = __halves2half2(h0, h1);
        *reinterpret_cast<__half2*>(bop + off + (uint32_t)N * 128u) = __halves2half2(l0, l1);
      }
    }
  }
}
// all consumer warps: make the generic-proxy writes of the B operand visible to the tensor cores (async proxy) and
// wait until every warp has written its part
template <int NTHREADS>
__device__ __forceinline__ void tc_publish_b() {
  fence_proxy_async();
  named_bar_sync(1, NTHREADS);
}

}  // namespace uis
