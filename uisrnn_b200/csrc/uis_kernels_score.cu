// score(): the neg_likelihood of given labellings (uis_score / uis_score_device in include/uisrnn_b200.h).
//
// With the labels fixed there is no search: the trace a forced decode would build visits every cluster's frames in
// order, and a cluster's state (running mean, hidden state) depends only on the frames it has seen.  So every
// (utterance, cluster) pair is an independent chain -- start from hidden0, one GRU + MLP step per visit, the
// off-by-one running mean -- and all chains of all utterances fill the columns of the FFMA weight pass (run_pass,
// uis_beam.cuh) densely.  Three kernels after the input projection:
//   uis_score_kernel     persistent, one CTA per SM, C::CP columns in flight per CTA, each bound to a chain pulled
//                        from a longest-first queue.  One weight pass advances every column by one visit; the new mean's
//                        Gaussian term against the chain's next frame goes to mse[row].  A chain of n frames needs n - 1
//                        passes (the state after its last visit is never scored).
//   score_first_kernel   mean0 against the first frame of every chain (one warp each).
//   score_reduce_kernel  one thread per utterance walks its frames: the transition / ddCRP term from the block counts,
//                        loss = fl32(f64(mse) - pen), and the fp32 running sum -- the arithmetic of the beam kernel's
//                        phases P1a / P1c.
// Pass and Gaussian term are the beam kernel's own functions, so a labelling that the FFMA beam search kept gets the
// same bits from both.
#include "uis_launch.cuh"

namespace uis {

// Shared memory of the chain kernel.  The weight ring and XA / XB are those of the beam kernel (make_layout);
// the rest is the column table.
template <int H, int D>
struct ScoreLayout {
  static constexpr int CP = BeamCP<H>::value;
  static constexpr unsigned ring = 0;
  static constexpr unsigned xa = ring + kStages * kStageBytes;
  static constexpr unsigned xb = xa + H * CP * 4;
  static constexpr unsigned wv = xb + H * CP * 4;
  static constexpr unsigned cols = wv + D * 4;                // collane, colsrc, colnew, colvis [CP] ints
  static constexpr unsigned colrow = cols + 4 * CP * 4;       // [CP] long long
  static constexpr unsigned cstart = colrow + CP * 8;         // [CP] long long: chain's first entry in chain_rows
  static constexpr unsigned cstate = cstart + CP * 8;         // chain, pos, len, cur, fresh [CP] ints
  static constexpr unsigned bars = (cstate + 5 * CP * 4 + 15) / 16 * 16;
  static constexpr unsigned misc = bars + 2 * kStages * 8;
  static constexpr unsigned phase = misc + 64;
  static constexpr unsigned total = phase + 16 * 8;
};

template <int H, int D, bool DEEP>
__global__ void __launch_bounds__(Cfg<H, D>::BLOCK, 1) uis_score_kernel(const __grid_constant__ ScoreParams sp) {
  using C = Cfg<H, D, BeamCP<H>::value>;
  using L = ScoreLayout<H, D>;
  constexpr int NT = C::NT, NW = C::NW, UPT = C::UPT, CP = C::CP;
  const BeamParams& p = sp.b;
  extern __shared__ __align__(128) unsigned char smem[];
  float* ring = reinterpret_cast<float*>(smem + L::ring);
  float* XA = reinterpret_cast<float*>(smem + L::xa);
  float* XB = reinterpret_cast<float*>(smem + L::xb);
  float* wv = reinterpret_cast<float*>(smem + L::wv);
  int* collane = reinterpret_cast<int*>(smem + L::cols);
  int* colsrc = collane + CP; int* colnew = collane + 2 * CP; int* colvis = collane + 3 * CP;
  long long* colrow = reinterpret_cast<long long*>(smem + L::colrow);
  long long* cstart = reinterpret_cast<long long*>(smem + L::cstart);
  int* cchain = reinterpret_cast<int*>(smem + L::cstate);
  int* cpos = cchain + CP; int* clen = cchain + 2 * CP; int* ccur = cchain + 3 * CP; int* cfresh = cchain + 4 * CP;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + L::bars);
  uint64_t* empty = full + kStages;
  volatile int* misc = reinterpret_cast<volatile int*>(smem + L::misc);
  long long* ph = reinterpret_cast<long long*>(smem + L::phase);  // run_pass's phase counters (thread 0)
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  // Weight-ring prologue.  The beam kernel's (uis_beam.cuh) also sets up the tensor-core, cluster and
  // stationary-weights engines; shared, it would branch on its caller, so this is the FFMA part of it.
  if (tid == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], NW);
    }
    for (int i = 0; i < 16; ++i) { misc[i] = 0; ph[i] = 0; }
    ph[10] = clock64();
    fence_mbar_init();
  }
  __syncthreads();
  if (warp >= NW) {  // producer warp (+ the idle warps of its warpgroup)
    if constexpr (C::REBALANCE) asm volatile("setmaxnreg.dec.sync.aligned.u32 24;");
    if (warp == NW && lane == 0) producer_loop<C>(p, ring, full, empty, misc);
    return;
  }
  if constexpr (C::REBALANCE) asm volatile("setmaxnreg.inc.sync.aligned.u32 240;");

  const int DH = p.depth * H;
  const size_t pool_m_stride = (size_t)2 * D, pool_h_stride = (size_t)2 * DH;  // column m: slots 2m, 2m + 1
  float* pool_mean_cta = p.pool_mean + (size_t)blockIdx.x * CP * pool_m_stride;
  float* pool_hidden_cta = p.pool_hidden + (size_t)blockIdx.x * CP * pool_h_stride;
  float bh[C::RG], b1r[UPT];
#pragma unroll
  for (int i = 0; i < C::RG; ++i) bh[i] = p.bhh[(i / UPT) * H + tid + NT * (i % UPT)];
#pragma unroll
  for (int u = 0; u < UPT; ++u) b1r[u] = p.b1[tid + NT * u];
  const float b2r = tid < D ? p.b2[tid] : 0.f;
  if (tid < D) wv[tid] = p.wvec[tid];
  long long st_cols = 0, st_pass = 0;  // thread 0's

  // (thread 0) bind column m to the next queued chain, or retire it (a device plan's count is read here, where it is
  // used: held across the loop it costs the larger shapes a spill; the surplus CTAs of its grid find the queue empty)
  auto bind = [&](int m) {
    const int q = atomicAdd(p.queue, 1);
    cchain[m] = -1;
    if (q < (sp.counts ? __ldg(sp.counts + 1) : sp.queued)) {
      cchain[m] = q; cpos[m] = 0; ccur[m] = 0; cfresh[m] = 1;
      cstart[m] = sp.chain_off[q];
      clen[m] = (int)(sp.chain_off[q + 1] - sp.chain_off[q]);
    }
  };
  // a freshly bound chain starts from hidden0 (every layer) in its column's current slot
  auto init_fresh = [&]() {
    for (int m = 0; m < CP; ++m)
      if (cfresh[m] && cchain[m] >= 0)
        for (int q = tid; q < DH; q += NT) pool_hidden_cta[m * pool_h_stride + (size_t)ccur[m] * DH + q] = p.hidden0[q];
  };
  if (tid == 0)
    for (int m = 0; m < CP; ++m) { cfresh[m] = 0; bind(m); }
  named_bar_sync(1, NT);
  init_fresh();

  const ColCtx cc{collane, colsrc, colnew, colvis, colrow};
  unsigned it = 0;  // weight-ring tile counter
  long long& tmark = ph[10];
  for (;;) {
    named_bar_sync(1, NT);  // column states and fresh slots are written
    if (tid == 0) {  // the pass's column list: every live chain, one visit each
      int M = 0;
      for (int m = 0; m < CP; ++m) {
        if (cchain[m] < 0) continue;
        collane[M] = m; colsrc[M] = ccur[m]; colnew[M] = ccur[m] ^ 1; colvis[M] = cpos[m];
        colrow[M] = sp.chain_rows[cstart[m] + cpos[m]];
        ++M;
      }
      misc[MI_MTOT] = M;
      if (M) {
        st_cols += M; st_pass += 1;
        __threadfence_block();
        misc[MI_PUBLISHED] = misc[MI_PUBLISHED] + 1;  // the producer streams one pass
      }
    }
    named_bar_sync(1, NT);
    const int M = misc[MI_MTOT];
    if (M == 0) break;
    // gather the source hidden states (layer 0), transposed: XA[k][m]
#pragma unroll
    for (int u = 0; u < UPT; ++u) {
      const int j = tid + NT * u;
#pragma unroll
      for (int c = 0; c < CP / 4; ++c) {
        float hv[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int m = 4 * c + q;
          hv[q] = (m < M) ? pool_hidden_cta[(size_t)collane[m] * pool_h_stride + (size_t)colsrc[m] * DH + j] : 0.f;
        }
        reinterpret_cast<float4*>(XA + (size_t)j * CP)[c] = make_float4(hv[0], hv[1], hv[2], hv[3]);
      }
    }
    named_bar_sync(1, NT);
    run_pass_any<C, DEEP>(p, ring, full, empty, it, XA, XB, cc, 0, M, pool_mean_cta, pool_hidden_cta, bh, b1r, b2r, tid,
                          lane, ph, tmark);
    named_bar_sync(1, NT);
    // Gaussian term of every new mean against its chain's next frame, one warp per column
    for (int i = warp; i < M; i += NW) {
      const int m = collane[i];
      const long long row = sp.chain_rows[cstart[m] + cpos[m] + 1];
      const float* mu = pool_mean_cta + m * pool_m_stride + (size_t)colnew[i] * D;
      float4 m4[1][(D + 127) / 128];
#pragma unroll
      for (int k = 0; k < (D + 127) / 128; ++k)
        if (lane * 4 + k * 128 < D) m4[0][k] = *reinterpret_cast<const float4*>(mu + lane * 4 + k * 128);
      const bool live[1] = {true};
      const float term = gauss_rows<D, 1>(m4, live, p.x + (size_t)row * D, wv, lane);
      if (lane == 0) sp.mse[row] = term;
    }
    named_bar_sync(1, NT);
    if (tid == 0)  // advance every column by one visit; a chain at its last frame hands its column on
      for (int i = 0; i < M; ++i) {
        const int m = collane[i];
        cfresh[m] = 0;
        cpos[m] += 1;
        ccur[m] ^= 1;
        if (cpos[m] == clen[m] - 1) bind(m);
      }
    named_bar_sync(1, NT);
    init_fresh();
  }
  if (tid == 0) {
    __threadfence_block();
    misc[MI_DONE] = 1;
    atomicAdd(&p.stats[0], (unsigned long long)st_cols);
    atomicAdd(&p.stats[1], (unsigned long long)st_pass);
  }
}

// mean0 against the first frame of every chain: one warp per chain (a device plan: the grid covers `chains` = rows
// warps, and those past the plan's chain count return).
template <int D>
__global__ void __launch_bounds__(256) score_first_kernel(const __grid_constant__ ScoreParams sp) {
  const BeamParams& p = sp.b;
  const int lane = threadIdx.x & 31;
  const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (w >= (sp.counts ? sp.counts[0] : sp.chains)) return;  // (whole warps)
  const long long row = sp.chain_rows[sp.chain_off[w]];
  float4 m4[1][(D + 127) / 128];
#pragma unroll
  for (int k = 0; k < (D + 127) / 128; ++k)
    if (lane * 4 + k * 128 < D) m4[0][k] = *reinterpret_cast<const float4*>(p.mean0 + lane * 4 + k * 128);
  const bool live[1] = {true};
  const float term = gauss_rows<D, 1>(m4, live, p.x + (size_t)row * D, p.wvec, lane);
  if (lane == 0) sp.mse[row] = term;
}

// One thread per utterance: loss_t = fl32(f64(mse_t) - pen_t) and S = fl32(S + loss_t) in frame order, with pen_t the
// beam kernel's transition / ddCRP term (phase P1a) of the trace so far under config `cfg`, whose totals go to row
// cfg of scores and increments to row cfg of frame_out.
__global__ void __launch_bounds__(128) score_reduce_kernel(const __grid_constant__ ScoreParams sp, int cfg) {
  const BeamParams& p = sp.b;
  const int u = blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= p.U) return;
  const JobLogs lg = job_logs(p, cfg);
  float* frame_out = sp.frame_out ? sp.frame_out + (size_t)cfg * sp.frame_stride : nullptr;
  const long long r0 = p.row_off[u], r1 = p.row_off[u + 1];
  int* blk = sp.blocks + r0;  // block counts of the utterance's clusters (K <= frames)
  int K = 0, last = -1, tot = 0;
  float S = 0.f;
  for (long long r = r0; r < r1; ++r) {
    const int c = sp.labels[r];
    const bool isnew = c >= K;
    double pen;
    if (!isnew) pen = (c == last) ? lg.log_1mp0 : (lg.log_p0 + __ldg(p.logn + blk[c])) - __ldg(lg.logtot + tot);
    else pen = (lg.log_p0 + lg.log_alpha) - __ldg(lg.logtot + tot);
    const float loss = __double2float_rn((double)sp.mse[r] - pen);
    S = __fadd_rn(S, loss);
    if (frame_out) frame_out[r] = loss;
    const bool moved = isnew || c != last;
    if (isnew) { blk[c] = 1; K += 1; }
    else if (moved) blk[c] += 1;
    tot += moved ? 1 : 0;
    last = c;
  }
  sp.scores[(size_t)cfg * sp.score_stride + u] = S;
}

unsigned score_smem(int H, int D) {
  unsigned smem = kNoKernel;
  with_shape(AllShapes{}, H, D, [&](auto s) { smem = ScoreLayout<decltype(s)::H, decltype(s)::D>::total; });
  return smem;
}

bool launch_score_chains(int H, int D, const ScoreParams& sp, int ctas, cudaStream_t st, cudaError_t* err) {
  return with_shape(AllShapes{}, H, D, [&](auto s) {
    using S = decltype(s);
    auto kern = sp.b.depth > 1 ? uis_score_kernel<S::H, S::D, true> : uis_score_kernel<S::H, S::D, false>;
    *err = launch_with_smem(kern, sp, ctas, Cfg<S::H, S::D>::BLOCK, ScoreLayout<S::H, S::D>::total, st);
  });
}

bool launch_score_first(int H, int D, const ScoreParams& sp, cudaStream_t st, cudaError_t* err) {
  const unsigned blocks = (unsigned)(((long long)sp.chains * 32 + 255) / 256);
  return with_shape(AllShapes{}, H, D, [&](auto s) {
    score_first_kernel<decltype(s)::D><<<blocks, 256, 0, st>>>(sp);
    *err = cudaGetLastError();
  });
}

cudaError_t launch_score_reduce(const ScoreParams& sp, int cfg, cudaStream_t st) {
  score_reduce_kernel<<<(sp.b.U + 127) / 128, 128, 0, st>>>(sp, cfg);
  return cudaGetLastError();
}

}  // namespace uis
