// Persistent beam-search kernel for UIS-RNN predict() on sm_90a  (look_ahead = 1, depth = 1).
//
// What it replaces (all under /root/reference/uisrnn/): the whole loop body of
// UISRNN.predict_single (uisrnn.py:529-561) -- _calculate_score (:455-477), the np.sort/argsort
// top-k (:546-552), _update_beam_state for the winners (:388-453), CoreRNN.forward (:45-52) and
// loss_func.weighted_mse_loss (loss_func.py:19-41) -- with BeamState (:55-77) kept on device.
//
// Mapping to the hardware
//   * one persistent CTA per SM.  A CTA runs G "lanes"; each lane pulls utterances (longest
//     first) from a global queue and runs ALL test_iteration*N beam steps of its utterance
//     without returning to the host.  Lanes only share the weight stream: one pass over the
//     weights serves the GRU columns of every lane's current step.
//   * per step the only heavy work is  h' = GRU(x_t, h_src),  mean = W2 relu(W1 h' + b1) + b2  for
//     the DISTINCT source states of the step's winners (M <= beam_size per lane): three skinny
//     (rows x 512) x (512 x M) products.  The fp32 weights (4.7 MB, L2-resident) are streamed
//     through a 4-stage shared-memory ring by a producer warp with 1-D TMA bulk copies
//     (cp.async.bulk + mbarrier complete_tx).  Consumer threads hold a register tile of
//     R rows x 16 columns (R = 6 for the GRU gates, 4 for the MLP layers with the K dimension
//     split over thread groups) so that each value fetched from shared memory feeds >= 3 FMAs:
//     the shared-memory return path (one 32-bit register per lane per cycle per SM) -- not
//     the FMA pipe -- is what bounds a skinny matvec batch otherwise.
//   * hypothesis state is a slot pool in global memory (L2): slot = (mean[D], hidden[H]) written
//     once and never modified; a hypothesis is a table of (slot, block count, visit count) per
//     cluster held in shared memory.  A child differs from its parent in ONE table entry, so the
//     re-pack after the top-k is an index shuffle plus M slot writes (BeamState copies in the
//     reference are shallow too, uisrnn.py:66-69).
//   * scoring needs no GRU at look_ahead 1 (uisrnn.py:411-414 uses the pre-update mean;
//     :438-443 uses the per-model constant CoreRNN(0, h0)), so candidates are scored first
//     (one warp per candidate, fp64 log terms from host-built tables), ranked by counting, and
//     only the winners' distinct source states go through the GRU.
#pragma once
#include "uis_common.cuh"
#include "uis_beam_tc.cuh"
#include "uis_beam_stat.cuh"

namespace uis {

constexpr int kStages = 2;              // weight ring depth
constexpr int kStageBytes = 48 * 1024;  // bytes per ring stage
constexpr int kInitSlot = 0;            // pool slot holding (mean0, hidden0)
#ifndef UIS_CP_BEAM
#define UIS_CP_BEAM 20
#endif
constexpr int kCPBeam = UIS_CP_BEAM;             // GRU columns per weight pass, look_ahead-1 kernel (two lanes need <= 20 in ~99 % of the steps)
// hidden sizes above 512: 8 columns per pass keep XA / XB (H x CP floats each) and the accumulator tile within budget
template <int H> struct BeamCP { static constexpr int value = H > 512 ? 8 : kCPBeam; };
template <int H> __host__ __device__ constexpr int beam_cp() { return BeamCP<H>::value; }
constexpr int kCPCluster = 12;          // cluster (latency) mode: one lane per cluster, <= 12 columns per pass
constexpr int kXchVals = 24;            // floats per thread and exchange round of the cluster K-split
constexpr int kCPTree = 16;             // look-ahead tree kernel (shared memory goes to the node arrays instead)
// hidden sizes above 512: at 16 columns the tree kernel's XA / XB alone would take 128 KB beside the 96 KB weight ring;
// 8 columns leave about the node capacity of (512, 256).  make_tree_layout, the kernel and the host's sizing use this.
template <int H> struct TreeCP { static constexpr int value = H > 512 ? 8 : kCPTree; };
template <int H> __host__ __device__ constexpr int tree_cp() { return TreeCP<H>::value; }
constexpr int kMaxLanes = 8;
constexpr int kMaxBeam = 128;  // beam_size served by the look_ahead-1 kernels (phase P3 walks the winners in chunks of 32)
constexpr int kMaxDepth = 4;             // stacked GRU layers supported on device

struct TabEntry {
  int slot;    // index into the lane's slot pool
  int blocks;  // block_counts[c]        (uisrnn.py:431-432, 451)
  int visits;  // #{trace == c}          (uisrnn.py:425-428)
  int pad;
};

struct SmemLayout {
  unsigned ring, xa, xb, wv, lanes, lane_stride, cols, bars, misc, phase, xch, xbar, slist, total;
  // offsets inside one lane block
  unsigned l_xt, l_tabs, l_meta, l_candoff, l_keys, l_svals, l_wins, l_wcol, l_lcol, l_used, l_scored, l_ls;
};

struct BeamParams {
  // model (device pointers)
  const float* whh_t;    // [H][3H]   = gru.weight_hh_l0 transposed (k-major)
  // stacked layers l = 1..depth-1 (nn.GRU feeds layer l with layer l-1's new hidden state):
  const float* wih_up_t[kMaxDepth - 1];  // [H][3H] = gru.weight_ih_l{l} transposed
  const float* whh_up_t[kMaxDepth - 1];  // [H][3H] = gru.weight_hh_l{l} transposed
  const float* bih_up;   // [depth-1][3H]
  const float* bhh_up;   // [depth-1][3H]
  int depth;
  const float* w1_t;     // [H][H]    = linear_mean1.weight transposed
  const float* w2_t;     // [H][D]    = linear_mean2.weight transposed
  const float* bhh;      // [3H]
  const float* b1;       // [H]
  const float* b2;       // [D]
  const float* wvec;     // [D]  1 / (2 sigma2)
  const float* mean0;    // [D]
  const float* hidden0;  // [depth][H]
  const double* logn;    // [>= maxTN + 2]  log(i)
  // Decoding parameters.  The kernels decode p.U jobs: job j is utterance j % n_utt under config j / n_utt (a call
  // without a sweep is one config holding the model's values, so job = utterance).
  const double* cfg_log;      // [configs][3]  log(p0), log(1 - p0), log(crp_alpha)
  const double* logtot;       // [configs][logtot_stride]  log(i + crp_alpha), i < logtot_stride (>= maxTN + 2)
  long long logtot_stride;
  int n_utt;                  // distinct utterances (rows, spk_bound); outputs are per job
  // inputs
  const float* x;           // [rows][D]
  const float* gi;          // [rows][3H]  W_ih x + b_ih
  const long long* row_off; // [n_utt + 1]
  const int* order;         // [U] job ids, longest utterance first, the configs of one utterance side by side
  int U, B, Kcap, T, P, maxN, G;
  int L, node_cap, leaf_cap, maxTN, maxSteps;  // look_ahead >= 2 (uis_beam_tree.cuh) only
  // tensor-core pass (uis_beam_tc.cuh): fp16 hi/lo weight planes [2 * (3H + H + D)][H] behind a tensor map
  alignas(64) CUtensorMap tc_wmap;
  float tc_sh, tc_sa;                  // power-of-two scales of the hidden columns and of a = relu(W1 h' + b1)
  float tc_inv_hh, tc_inv_1, tc_inv_2; // 1 / (weight scale * operand scale) per matrix
  float* tc_scratch;                   // [ctas][N][H]  a = relu(W1 h' + b1) between the W1 and the W2 product
  SmemLayout tc_layout;                // make_layout() of the launched instantiation (no registers held for it)
  // stationary-weights mode (uis_beam_stat.cuh)
  unsigned* stat_bar;                  // [groups][32]: word 0 of a group = arrival counter of its barrier (zero at launch; one 128-byte line per group)
  float* stat_scratch;                 // [groups][kCPCluster][H]  a = relu(W1 h' + b1), exchanged through L2
  // per-(CTA, lane) workspace
  float* pool_mean;    // [ctas*G][P][D]
  float* pool_hidden;  // [ctas*G][P][depth][H]
  float* pool_mse;     // [ctas*G][P]  Gaussian term of the slot's mean against the lane's current frame
  unsigned* bp;        // [ctas*G][maxN][B]  (parent << 16) | cluster
  int* queue;          // [1] next position in `order`
  // outputs
  int* labels;  // [rows]
  int* status;  // [U]   0 ok, -4 overflow
  unsigned long long* stats;  // [8]
  // debug taps (device buffers, may be null)
  int trace_utt;
  int trace_capacity;
  int* dbg_win;            // [cap][2]
  float* dbg_score;        // [cap]
  long long* dbg_off;      // [steps + 1]
  float* dbg_final_scores; // [U][B]
  int* dbg_final_k;        // [U]
  float* dbg_best_mean;    // [Kcap][D]
  float* dbg_best_hidden;  // [Kcap][depth][H]
  int* dbg_best_blocks;    // [Kcap]
  // look-ahead spill kernel (uis_beam_tree.cuh, SPILL = true); these fit the struct's tail padding (sizeof stays 768)
  unsigned char* tree_arena;  // [ctas][make_tree_arena(node_cap, leaf_cap, P).total]
  int tree_spill_all;         // 1: decode every utterance, not only those the shared-memory kernel left at status -5
  // speaker bounds (uis_predict*_bounded), indexed by utterance id; null = unbounded
  const int* spk_bound;  // [U][2]: max_speakers (0 = none), min_speakers
  int* spk_out;          // [U]    clusters of the returned hypothesis, 0 for a failed utterance
  // N-best output (uis_predict*_nbest): hypothesis j of utterance u is the j-th final rank with at least
  // min_speakers clusters (nbest_rank); its labels are plane j of `labels` (plane stride label_plane rows)
  int n_best;              // >= 1; 1 = labels plane 0 only
  long long label_plane;   // rows per label plane (n_best > 1)
  float* nbest_scores;     // [U][n_best]  neg_likelihood, +inf where absent (may be null)
  int* nbest_speakers;     // [U][n_best]  clusters, 0 where absent (may be null)
  int* nbest_count;        // [U]          hypotheses returned (may be null)
};

// The log terms of a job's config (uisrnn.py:416-418, 445): the transition / ddCRP penalty of a candidate is
//   existing cluster c: (c == last) ? log_1mp0 : (log_p0 + logn[blocks_c]) - logtot[tot]
//   new cluster:        (log_p0 + log_alpha) - logtot[tot]
struct JobLogs {
  double log_p0, log_1mp0, log_alpha;
  const double* logtot;
};
__device__ inline JobLogs job_logs(const BeamParams& p, int cfg) {
  const double* v = p.cfg_log + 3 * cfg;
  return JobLogs{__ldg(v), __ldg(v + 1), __ldg(v + 2), p.logtot + (size_t)cfg * p.logtot_stride};
}

// Per-utterance speaker bounds: a hypothesis may hold at most spk_max clusters; the returned one is the best-ranked
// final hypothesis with at least spk_min clusters (rank 0 if there is none).
__device__ inline int spk_max(const BeamParams& p, int u) {
  const int v = p.spk_bound ? p.spk_bound[2 * u] : 0;
  return v > 0 ? v : 0x7fffffff;
}
__device__ inline int spk_min(const BeamParams& p, int u) { return p.spk_bound ? p.spk_bound[2 * u + 1] : 0; }
// First rank r < n with K[r] >= kmin, else 0.
__device__ inline int spk_pick(const int* K, int n, int kmin) {
#pragma unroll 1
  for (int r = 0; r < n; ++r)
    if (K[r] >= kmin) return r;
  return 0;
}
// Rank of N-best hypothesis j < n_best among n final ranks: the j-th rank with K[r] >= kmin; rank 0 for j = 0 when
// none qualifies (spk_pick); -1 when absent.
__device__ inline int nbest_rank(const int* K, int n, int kmin, int j) {
  int seen = 0;
#pragma unroll 1
  for (int r = 0; r < n; ++r)
    if (K[r] >= kmin && seen++ == j) return r;
  return (j == 0) ? 0 : -1;
}
// Hypotheses an N-best call returns: the qualifying ranks up to n_best, or 1 (the rank-0 fall-back).
__device__ inline int nbest_n(const int* K, int n, int kmin, int n_best) {
  int c = 0;
#pragma unroll 1
  for (int r = 0; r < n && c < n_best; ++r) c += K[r] >= kmin;
  return c > 0 ? c : 1;
}
// Per-hypothesis outputs of hypothesis j (rank r, -1 = absent) of a finished utterance u.
__device__ inline void nbest_store(const BeamParams& p, int u, int j, int r, const int* K, const float* Nl) {
  const float INF = __int_as_float(0x7f800000);
  if (p.nbest_scores) p.nbest_scores[(size_t)u * p.n_best + j] = r >= 0 ? Nl[r] : INF;
  if (p.nbest_speakers) p.nbest_speakers[(size_t)u * p.n_best + j] = r >= 0 ? K[r] : 0;
}

template <int V> struct Pow2Floor { static constexpr int value = (V >= 2) ? 2 * Pow2Floor<V / 2>::value : 1; };
template <> struct Pow2Floor<1> { static constexpr int value = 1; };
template <> struct Pow2Floor<0> { static constexpr int value = 1; };
constexpr int cmin(int a, int b) { return a < b ? a : b; }

template <int H_, int D_, int CP_ = kCPBeam>
struct Cfg {
  static constexpr int H = H_, D = D_;
  static constexpr int CP = CP_;                  // columns per weight pass = row stride of XA / XB
  static constexpr int UPT = (H >= 512) ? 2 : 1;  // hidden units per consumer thread
  static constexpr int NT = H / UPT;              // consumer threads
  static constexpr int NW = NT / 32;
  // Register re-balancing (setmaxnreg): with 8 consumer warps the launch allocation caps every
  // thread at 168 registers; a 4-warp producer group that shrinks itself to 24 registers lets
  // the two consumer warpgroups grow to 240 (6x16 accumulator tile + operand double-buffering
  // without spills).  Small configs (NT < 256) already have 255 registers per thread.
  static constexpr bool REBALANCE = (NT == 256);
  static constexpr int PRODUCER_THREADS = REBALANCE ? 128 : 32;
  static constexpr int BLOCK = NT + PRODUCER_THREADS;
  static constexpr int RG = 3 * UPT;              // GRU pass: rows per thread
  static constexpr int KG1 = UPT, TG1 = NT / KG1, R1 = H / TG1;             // W1 pass: K-groups, rows/thread
  static constexpr int R2 = (UPT == 2) ? 4 : 1, KG2 = NT * R2 / D, TG2 = NT / KG2;  // W2 pass
  static constexpr int KT_HH = Pow2Floor<kStageBytes / (12 * H)>::value;  // k-rows per ring stage
  static constexpr int KT_1 = cmin(Pow2Floor<kStageBytes / (4 * H)>::value, H);
  static constexpr int KT_2 = cmin(Pow2Floor<kStageBytes / (4 * D)>::value, H);
  static constexpr int N_HH = H / KT_HH, N_1 = H / KT_1, N_2 = H / KT_2;
  static constexpr int TILES_PER_PASS = N_HH + N_1 + N_2;
  static_assert(H % KT_HH == 0 && H % KT_1 == 0 && H % KT_2 == 0, "tile split");
  static_assert(KT_1 % KG1 == 0 && KT_2 % KG2 == 0, "K split");
  static_assert(TG2 * R2 == D && TG1 * R1 == H, "row split");
  static_assert(KG1 * H <= 2 * H && KG2 * D <= 2 * H, "K-split scratch must fit in XA+XB");
  static_assert(D % 4 == 0 && NT % 32 == 0 && D <= NT, "shape");
};

__host__ __device__ inline unsigned align_up(unsigned v, unsigned a) { return (v + a - 1) / a * a; }

// lane scalars (ints) ------------------------------------------------------------------------
enum { LS_U = 0, LS_N, LS_TN, LS_T, LS_NB, LS_GEN, LS_ACTIVE, LS_FAILED, LS_TRACED, LS_NFINITE, LS_KMAX,
       LS_NWIN, LS_ERR, LS_M, LS_COLBASE, LS_NE, LS_ROW0_LO, LS_ROW0_HI, LS_DBGROWS_LO, LS_DBGROWS_HI,
       LS_FRESH, LS_KHI, LS_KLO, LS_NLIST, LS_COUNT = 24 };  // LS_KHI / LS_KLO: speaker bounds; LS_NLIST: slots listed for scoring
// CTA scalars
enum { MI_PUBLISHED = 0, MI_DONE, MI_MTOT, MI_QNEXT, MI_MAXK };

template <int H, int D, int kCP = kCPBeam, bool XCL = false, int TCN = 0, bool STAT = false>
__host__ __device__ inline SmemLayout make_layout(int B, int Kcap, int G) {
  SmemLayout L;
  unsigned o = 0;
  if constexpr (TCN > 0) {  // tensor-core pass: ring of 16 KB weight boxes, B operand (both 1024-byte aligned)
    using TC = TcCfg<H, D, TCN>;
    L.ring = o;  o += TC::STAGES * kTcBoxBytes;
    L.xa = o;    o += TC::BOP_BYTES;
    L.xb = o;
  } else {
    L.ring = o;  o += STAT ? align_up(StatCfg<H, D>::BYTES, 128) : kStages * kStageBytes;  // STAT: the resident weight rows
    L.xa = o;    o += H * kCP * 4;
    L.xb = o;    o += H * kCP * 4;
  }
  L.wv = o;    o += D * 4;
  // ---- one lane block
  unsigned q = 0;
  L.l_xt = q;      q += 2 * D * 4;
  L.l_tabs = q;    q += 2u * B * Kcap * 16;
  L.l_meta = q;    q += 2u * 4 * B * 4;  // K,last,tot,nl  x2 generations
  L.l_candoff = q; q += align_up((B + 1) * 4, 16);
  const unsigned ne = (unsigned)B * (Kcap + 1);
  L.l_keys = q;    q += align_up(ne * 8, 16);
  L.l_svals = q;   q += align_up(ne * 4, 16);
  L.l_wins = q;    q += align_up(3u * B * 4, 16);
  L.l_wcol = q;    q += align_up((unsigned)B * 4, 16);
  L.l_lcol = q;    q += align_up(2u * B * 4, 16);  // lane-local column -> (source slot, new slot)
  const unsigned pw = ((unsigned)B * Kcap + B + 1 + 31) / 32;
  L.l_used = q;    q += align_up(pw * 4, 16);
  L.l_scored = q;  q += align_up(pw * 4, 16);  // slots whose Gaussian term against the current frame is in pool_mse
  L.l_ls = q;      q += LS_COUNT * 4;
  L.lane_stride = align_up(q, 16);
  L.lanes = o;     o += L.lane_stride * G;
  L.cols = o;      o += align_up(6u * G * B * 4, 16);  // collane, colsrc, colnew, colvis, colrow (8 B each)
  L.bars = o;
  if constexpr (TCN > 0) o += 2 * TcCfg<H, D, TCN>::STAGES * 8;  // full, empty
  else o += 2 * kStages * 8;
  L.misc = o;      o += 64;
  L.slist = o;     o += 4u * 64u * G;  // per lane: 64-entry slot list of the per-slot scoring
  L.phase = o;     o += 128 + 32;  // thread 0's statistics: 10 phase cycle counters, phase mark, 5 counters, 4 tensor-core pass counters
  L.xch = o; L.xbar = o;
  if (XCL) {  // cluster K-split: two exchange buffers of kXchVals floats per consumer thread + 2 mbarriers
    o = align_up(o, 16);
    L.xch = o;   o += 2u * kXchVals * (H / ((H >= 512) ? 2 : 1)) * 4;
    L.xbar = o;  o += 16;
  }
  if (TCN > 0) o += 1024;  // slack: the kernel aligns its dynamic shared memory to 1024 bytes (swizzle atoms)
  L.total = o;
  return L;
}

// ------------------------------------------------------------------ producer (one thread)
template <class C, bool XCL = false>
__device__ void producer_loop(const BeamParams& p, float* ring, uint64_t* full, uint64_t* empty,
                              volatile int* misc) {
  constexpr int H = C::H, D = C::D;
  // cluster mode: CTA `rank` of the cluster streams (and multiplies) only its share of the k-tiles of every
  // matrix -- the k-major layouts split contiguously
  const int xrank = XCL ? (int)cluster_ctarank() : 0, xsize = XCL ? (int)cluster_nctarank() : 1;
  unsigned it = 0;
  int pass = 0;
  for (;;) {
    while (misc[MI_PUBLISHED] <= pass) {
      if (misc[MI_DONE]) return;
      __nanosleep(64);
    }
    __threadfence_block();
    const int ngru = 1 + 2 * (p.depth - 1);  // W_hh_0, then (W_ih_l, W_hh_l) for every upper layer
    for (int seg = 0; seg < ngru + 2; ++seg) {
      const float* src;
      if (seg == 0) src = p.whh_t;
      else if (seg < ngru) src = ((seg - 1) & 1) ? p.whh_up_t[(seg - 1) / 2] : p.wih_up_t[(seg - 1) / 2];
      else src = (seg == ngru) ? p.w1_t : p.w2_t;
      const int ntiles = seg < ngru ? C::N_HH : (seg == ngru ? C::N_1 : C::N_2);
      const unsigned bytes = seg < ngru ? C::KT_HH * 3 * H * 4 : (seg == ngru ? C::KT_1 * H * 4 : C::KT_2 * D * 4);
      const int tcnt = ntiles / xsize, tbeg = xrank * tcnt;
      for (int t = tbeg; t < tbeg + tcnt; ++t, ++it) {
        const unsigned s = it % kStages, ph = (it / kStages) & 1;
        mbar_wait_parked(&empty[s], ph ^ 1);
        mbar_arrive_expect_tx(&full[s], bytes);
        tma_bulk_g2s(reinterpret_cast<char*>(ring) + (size_t)s * kStageBytes,
                     reinterpret_cast<const char*>(src) + (size_t)t * bytes, bytes, &full[s]);
      }
    }
    ++pass;
  }
}

// Consume one full weight pass without computing (a step with no winner at all), so that the
// producer, which was already told about the pass, never blocks on a full ring.
template <class C>
__device__ __forceinline__ void drain_pass(uint64_t* full, uint64_t* empty, unsigned& it, int lane, int depth = 1,
                                           int xsize = 1) {
  const int tiles = (C::TILES_PER_PASS + 2 * (depth - 1) * C::N_HH) / xsize;
  for (int t = 0; t < tiles; ++t, ++it) {
    const unsigned s = it % kStages, ph = (it / kStages) & 1;
    mbar_wait(&full[s], ph);
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[s]);
  }
}

// ------------------------------------------------------------------ consumer: one weight matrix
// acc[i][m] += sum_k Wt[k][tl + TG*i] * X[k][m]   for this thread's R rows and its K-group's
// share (KT/KG k-rows) of every ring tile.  Wt tiles are [KT][ROWS] floats; X is [H][C::CP].
// The operand loads are software-pipelined ACROSS ring tiles: the first k-step of tile t+1 is
// fetched (after its full-barrier test) before the last k-step of tile t is multiplied, so the
// mbarrier round trip and the shared-memory latency are not exposed at every tile boundary.
template <int R, int NC>
struct Operands {
  float w[R];
  float4 x[NC];
};

template <class C, int ROWS, int KT, int KG, int R, int NC, bool ZERO = true, bool XCL = false>
__device__ __forceinline__ void lin_pass(const float* __restrict__ ring, uint64_t* full, uint64_t* empty,
                                         unsigned& it, const float* __restrict__ X, float (&acc)[R][4 * NC],
                                         int tid, int lane, int xrank = 0, int xsize = 1) {
  constexpr int TG = C::NT / KG;
  constexpr int KPG = KT / KG;
  constexpr int NTILES_ALL = C::H / KT;
  // cluster mode: this CTA multiplies tiles [TILE0, TILE0 + NTILES) only (a partial sum over k)
  const int NTILES = XCL ? NTILES_ALL / xsize : NTILES_ALL;
  const int TILE0 = XCL ? xrank * NTILES : 0;
  const int kg = tid / TG, tl = tid % TG;
  if constexpr (ZERO) {
#pragma unroll
    for (int i = 0; i < R; ++i)
#pragma unroll
      for (int m = 0; m < 4 * NC; ++m) acc[i][m] = 0.f;
  }

  auto tile_w = [&](unsigned itx) -> const float* {
    return ring + (size_t)(itx % kStages) * (kStageBytes / 4) + (size_t)(kg * KPG) * ROWS + tl;
  };
  auto tile_x = [&](int tile) -> const float4* {
    return reinterpret_cast<const float4*>(X + (size_t)(tile * KT + kg * KPG) * C::CP);
  };
  // volatile ld.shared: keeps the loads of k-step s+1 AHEAD of the FFMAs of k-step s in the
  // instruction stream (the compiler otherwise sinks them next to their first use, which
  // exposes the ~30-cycle shared-memory latency with only 2 warps per scheduler)
  auto load = [&](Operands<R, NC>& o, const float* wt, const float4* xp, int kq) {
    const uint32_t wa = smem_u32(wt) + (uint32_t)(kq * ROWS) * 4u;
    const uint32_t xa = smem_u32(xp) + (uint32_t)(kq * (C::CP / 4)) * 16u;
#pragma unroll
    for (int i = 0; i < R; ++i)
      asm volatile("ld.shared.f32 %0, [%1];" : "=f"(o.w[i]) : "r"(wa + (uint32_t)(TG * i) * 4u));
#pragma unroll
    for (int c = 0; c < NC; ++c)
      asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];"
                   : "=f"(o.x[c].x), "=f"(o.x[c].y), "=f"(o.x[c].z), "=f"(o.x[c].w)
                   : "r"(xa + (uint32_t)c * 16u));
  };
  auto mac = [&](const Operands<R, NC>& o) {
#pragma unroll
    for (int c = 0; c < NC; ++c) {
#pragma unroll
      for (int i = 0; i < R; ++i) {  // IEEE-RN fmas, w broadcast over the 4 columns
        acc[i][4 * c + 0] = __fmaf_rn(o.x[c].x, o.w[i], acc[i][4 * c + 0]);
        acc[i][4 * c + 1] = __fmaf_rn(o.x[c].y, o.w[i], acc[i][4 * c + 1]);
        acc[i][4 * c + 2] = __fmaf_rn(o.x[c].z, o.w[i], acc[i][4 * c + 2]);
        acc[i][4 * c + 3] = __fmaf_rn(o.x[c].w, o.w[i], acc[i][4 * c + 3]);
      }
    }
  };

  Operands<R, NC> cur, nxt;
  mbar_wait(&full[it % kStages], (it / kStages) & 1);
  const float* wt = tile_w(it);
  const float4* xp = tile_x(TILE0);
  load(cur, wt, xp, 0);
  for (int tile = 0; tile < NTILES; ++tile) {
    const unsigned s = it % kStages;
#pragma unroll
    for (int kq = 0; kq < KPG; ++kq) {
      if (kq + 1 < KPG) {
        load(nxt, wt, xp, kq + 1);
      } else if (tile + 1 < NTILES) {
        const unsigned itn = it + 1;
        mbar_wait(&full[itn % kStages], (itn / kStages) & 1);
        wt = tile_w(itn);
        xp = tile_x(TILE0 + tile + 1);
        load(nxt, wt, xp, 0);
      }
      mac(cur);
      cur = nxt;
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[s]);
    ++it;
  }
}

// Sum the K-groups' partial results through shared memory.  On return out[q][m] holds the full
// sum for row tid + NT*q (q < RF).  `scratch` = XA..XB (2*H*C::CP floats), dead at this point.
template <class C, int ROWS, int KG, int R, int RF, int NC>
__device__ __forceinline__ void ksplit_reduce(float (&acc)[R][4 * NC], float* __restrict__ scratch,
                                              float (&out)[RF][4 * NC], int tid) {
  if constexpr (KG == 1) {
    static_assert(R == RF, "direct mapping");
#pragma unroll
    for (int q = 0; q < RF; ++q)
#pragma unroll
      for (int m = 0; m < 4 * NC; ++m) out[q][m] = acc[q][m];
  } else {
    constexpr int TG = C::NT / KG;
    const int kg = tid / TG, tl = tid % TG;
    named_bar_sync(1, C::NT);  // every thread is done reading the pass input
#pragma unroll
    for (int i = 0; i < R; ++i)
#pragma unroll
      for (int c = 0; c < NC; ++c)
        reinterpret_cast<float4*>(scratch + ((size_t)kg * ROWS + tl + TG * i) * C::CP)[c] =
            make_float4(acc[i][4 * c + 0], acc[i][4 * c + 1], acc[i][4 * c + 2], acc[i][4 * c + 3]);
    named_bar_sync(1, C::NT);
#pragma unroll
    for (int q = 0; q < RF; ++q) {
      const int row = tid + C::NT * q;
#pragma unroll
      for (int c = 0; c < NC; ++c) {
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (row < ROWS) {
          v = reinterpret_cast<const float4*>(scratch + (size_t)row * C::CP)[c];
#pragma unroll
          for (int g = 1; g < KG; ++g) {
            const float4 o = reinterpret_cast<const float4*>(scratch + ((size_t)g * ROWS + row) * C::CP)[c];
            v.x = __fadd_rn(v.x, o.x); v.y = __fadd_rn(v.y, o.y); v.z = __fadd_rn(v.z, o.z); v.w = __fadd_rn(v.w, o.w);
          }
        }
        out[q][4 * c + 0] = v.x; out[q][4 * c + 1] = v.y; out[q][4 * c + 2] = v.z; out[q][4 * c + 3] = v.w;
      }
    }
    named_bar_sync(1, C::NT);  // scratch may be overwritten by the caller from here on
  }
}

// Cluster K-split: all-reduce of NV floats per consumer thread across the CTAs of the cluster, through
// distributed shared memory.  Every CTA parks its partial values in its own buffer (double-buffered by the
// exchange count), tells every peer "ready" with a release-arrive on the PEER's mbarrier, waits until all
// peers have told it the same, and sums the partials of ranks 0, 1, ... in that order -- the same order in
// every CTA, so the replicas stay bit-identical.  A buffer is rewritten two exchanges later, after the next
// handshake, by which time every peer has consumed it (in-order issue: the adds below wait for the loads).
struct XchCtx {
  float* buf;      // [2][kXchVals][NT]
  uint64_t* bar;   // [2]
  unsigned rank, size, count;  // count = exchanges done so far (identical in every thread of the cluster)
};
template <int NT, int NV>
__device__ __forceinline__ void xch_allreduce(XchCtx& x, float (&v)[NV], int tid) {
  static_assert(NV <= kXchVals && NV % 4 == 0, "exchange round: a multiple of 4, at most kXchVals floats");
  const unsigned b = x.count & 1u, parity = (x.count >> 1) & 1u;
  float4* mine = reinterpret_cast<float4*>(x.buf + (size_t)b * kXchVals * NT);  // [NV / 4][NT] float4
#pragma unroll
  for (int i = 0; i < NV / 4; ++i) mine[i * NT + tid] = make_float4(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
  named_bar_sync(1, NT);
  if (tid == 0)
    for (unsigned r = 0; r < x.size; ++r)
      if (r != x.rank) mbar_arrive_remote(dsmem_addr(smem_u32(&x.bar[b]), r));
  mbar_wait_cluster(&x.bar[b], parity);
  const uint32_t base = smem_u32(mine + tid);
  float sum[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) sum[i] = 0.f;
  for (unsigned r = 0; r < x.size; ++r) {
    if (r == x.rank) {
#pragma unroll
      for (int i = 0; i < NV; ++i) sum[i] = (r == 0) ? v[i] : __fadd_rn(sum[i], v[i]);
    } else {
      const uint32_t ra = dsmem_addr(base, r);
      float4 t[NV / 4];
#pragma unroll
      for (int i = 0; i < NV / 4; ++i) t[i] = dsmem_ld_f32x4(ra + (uint32_t)(i * NT) * 16u);  // 16 B per thread and load
#pragma unroll
      for (int i = 0; i < NV / 4; ++i) {
        sum[4 * i + 0] = (r == 0) ? t[i].x : __fadd_rn(sum[4 * i + 0], t[i].x);
        sum[4 * i + 1] = (r == 0) ? t[i].y : __fadd_rn(sum[4 * i + 1], t[i].y);
        sum[4 * i + 2] = (r == 0) ? t[i].z : __fadd_rn(sum[4 * i + 2], t[i].z);
        sum[4 * i + 3] = (r == 0) ? t[i].w : __fadd_rn(sum[4 * i + 3], t[i].w);
      }
    }
  }
#pragma unroll
  for (int i = 0; i < NV; ++i) v[i] = sum[i];
  x.count += 1;
}
// handshake without data: nobody leaves (and frees its shared memory) while a peer may still read it
template <int NT>
__device__ __forceinline__ void xch_barrier(XchCtx& x, int tid) {
  const unsigned b = x.count & 1u, parity = (x.count >> 1) & 1u;
  named_bar_sync(1, NT);
  if (tid == 0)
    for (unsigned r = 0; r < x.size; ++r)
      if (r != x.rank) mbar_arrive_remote(dsmem_addr(smem_u32(&x.bar[b]), r));
  mbar_wait_cluster(&x.bar[b], parity);
  x.count += 1;
}

// weighted_mse_loss (loss_func.py:33-41) of NB mean rows against one frame, by one warp: sum_d fl(fl(diff^2) * w_d)
// in fp32, lane l taking d = 4 l + 128 i in that order, then a butterfly over the lanes (xor 16, 8, 4, 2, 1); divided
// by the count of rows whose first squared difference is non-zero (0 -> inf / nan).  m4[q] holds row q's values at the
// lane's positions (rows with live[q] false are skipped and give 0); xs and wv point at the frame and the weights
// 1 / (2 sigma2).  Lane q < NB returns row q's term, the other lanes row 0's (the tails run side by side).  The beam
// kernels and the chain kernel of score() both call this, so a slot's term against a frame has the same bits in both.
template <int D, int NB>
__device__ __forceinline__ float gauss_rows(const float4 (&m4)[NB][(D + 127) / 128], const bool (&live)[NB],
                                            const float* xs, const float* wv, int lane) {
  float acc[NB], d0sq[NB];
#pragma unroll
  for (int q = 0; q < NB; ++q) {
    acc[q] = 0.f; d0sq[q] = 1.f;
#pragma unroll
    for (int i = 0; i < (D + 127) / 128; ++i) {
      const int d = lane * 4 + i * 128;
      if (d < D && live[q]) {
        const float4 x4 = *reinterpret_cast<const float4*>(xs + d);
        const float4 w4 = *reinterpret_cast<const float4*>(wv + d);
        const float e0 = __fsub_rn(m4[q][i].x, x4.x), e1 = __fsub_rn(m4[q][i].y, x4.y);
        const float e2 = __fsub_rn(m4[q][i].z, x4.z), e3 = __fsub_rn(m4[q][i].w, x4.w);
        const float q0 = __fmul_rn(e0, e0);
        if (d == 0) d0sq[q] = q0;
        acc[q] = __fadd_rn(acc[q], __fmul_rn(q0, w4.x));
        acc[q] = __fadd_rn(acc[q], __fmul_rn(__fmul_rn(e1, e1), w4.y));
        acc[q] = __fadd_rn(acc[q], __fmul_rn(__fmul_rn(e2, e2), w4.z));
        acc[q] = __fadd_rn(acc[q], __fmul_rn(__fmul_rn(e3, e3), w4.w));
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {  // interleaved butterfly reductions
#pragma unroll
    for (int q = 0; q < NB; ++q) acc[q] = __fadd_rn(acc[q], __shfl_xor_sync(0xffffffffu, acc[q], o));
  }
  float my_acc = acc[0], my_d0 = __shfl_sync(0xffffffffu, d0sq[0], 0);
#pragma unroll
  for (int q = 1; q < NB; ++q) {
    const float dq = __shfl_sync(0xffffffffu, d0sq[q], 0);
    if (lane == q) { my_acc = acc[q]; my_d0 = dq; }
  }
  if (my_d0 == 0.f) my_acc = __fdiv_rn(my_acc, 0.f);  // zero "non-zero rows" (loss_func.py:36)
  return my_acc;
}

// Per-column context of the current weight pass (shared memory, written in phase P4).
struct ColCtx {
  const int* lane;  // [Mtot] lane of the column
  const int* src;   // source slot
  const int* dst;   // new slot
  const int* vis;   // visits of the source entry BEFORE this update
  const long long* girow;  // row of p.gi (= W_ih x + b_ih, written by input_proj_kernel) of the column's frame
};

// ---- one full weight pass (GRU -> W1 -> W2) for columns [m0, m0 + Mp) -----------------------
template <class C, int NC, bool DEEP, bool XCL = false>
__device__ __forceinline__ void run_pass(const BeamParams& p, const float* ring, uint64_t* full, uint64_t* empty,
                                         unsigned& it, float* XA, float* XB,
                                         const ColCtx cc, int m0, int Mp, float* pool_mean_cta,
                                         float* pool_hidden_cta, const float (&bh)[C::RG], const float (&b1r)[C::UPT],
                                         float b2r, int tid, int lane, long long* ph, long long& tmark,
                                         XchCtx* xc = nullptr) {
  const int xrank = XCL ? (int)xc->rank : 0, xsize = XCL ? (int)xc->size : 1;
  constexpr int H = C::H, D = C::D, NT = C::NT, UPT = C::UPT;
  const int DH = p.depth * H;
  const size_t lane_pool_h = (size_t)p.P * DH, lane_pool_m = (size_t)p.P * D;
  // ---------------- GRU gates: acc[g*UPT + u][m] = (W_h{r,z,n} h_src)[unit tid + NT*u]
  {
    float acc[C::RG][4 * NC];
    lin_pass<C, 3 * H, C::KT_HH, 1, C::RG, NC, true, XCL>(ring, full, empty, it, XA, acc, tid, lane, xrank, xsize);
    if constexpr (XCL) {  // partial sums over this CTA's k-tiles -> full sums, one 4-column group per round
      static_assert(!DEEP && 4 * C::RG <= kXchVals, "cluster mode: depth 1");
#pragma unroll
      for (int c = 0; c < NC; ++c) {
        float v[4 * C::RG];
#pragma unroll
        for (int i = 0; i < C::RG; ++i)
#pragma unroll
          for (int q = 0; q < 4; ++q) v[4 * i + q] = acc[i][4 * c + q];
        xch_allreduce<NT, 4 * C::RG>(*xc, v, tid);
#pragma unroll
        for (int i = 0; i < C::RG; ++i)
#pragma unroll
          for (int q = 0; q < 4; ++q) acc[i][4 * c + q] = v[4 * i + q];
      }
    }
    // GRU cell, PyTorch gate order r,z,n (uisrnn.py:39-47):  h' = (h - n) * z + n
#pragma unroll
    for (int u = 0; u < UPT; ++u) {
      const int j = tid + NT * u;
#pragma unroll
      for (int c = 0; c < NC; ++c) {
        const float4 hold = reinterpret_cast<const float4*>(XA + (size_t)j * C::CP)[c];
        const float ho[4] = {hold.x, hold.y, hold.z, hold.w};
        float hn[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int m = 4 * c + q;
          hn[q] = 0.f;
          if (m < Mp) {
            const float* gi = p.gi + (size_t)cc.girow[m0 + m] * 3 * H;  // L2-resident, re-read per column (L1 hit)
            const float r = sigmoid_f32(__fadd_rn(gi[j], __fadd_rn(acc[0 * UPT + u][m], bh[0 * UPT + u])));
            const float z = sigmoid_f32(__fadd_rn(gi[H + j], __fadd_rn(acc[1 * UPT + u][m], bh[1 * UPT + u])));
            const float n = tanhf(__fadd_rn(gi[2 * H + j], __fmul_rn(r, __fadd_rn(acc[2 * UPT + u][m], bh[2 * UPT + u]))));
            hn[q] = __fadd_rn(__fmul_rn(__fsub_rn(ho[q], n), z), n);
            pool_hidden_cta[(size_t)cc.lane[m0 + m] * lane_pool_h + (size_t)cc.dst[m0 + m] * DH + j] = hn[q];
          }
        }
        reinterpret_cast<float4*>(XB + (size_t)j * C::CP)[c] = make_float4(hn[0], hn[1], hn[2], hn[3]);
      }
    }
  }
  // ---------------- stacked layers (nn.GRU depth >= 2, eval mode: no inter-layer dropout):
  //   layer l sees x = h'_{l-1} (in XB) and its own previous state h_l (gathered into XA)
  if constexpr (DEEP)
  for (int l = 1; l < p.depth; ++l) {
    named_bar_sync(1, NT);
    float acc[C::RG][4 * NC];
    lin_pass<C, 3 * H, C::KT_HH, 1, C::RG, NC>(ring, full, empty, it, XB, acc, tid, lane);  // W_ih_l h'_{l-1}
    float ni[UPT][4 * NC];  // input part of the candidate gate stays separate: n = tanh(i_n + r * h_n)
#pragma unroll
    for (int u = 0; u < UPT; ++u)
#pragma unroll
      for (int m = 0; m < 4 * NC; ++m) { ni[u][m] = acc[2 * UPT + u][m]; acc[2 * UPT + u][m] = 0.f; }
    named_bar_sync(1, NT);  // every thread is done with XA (layer l-1) ...
#pragma unroll
    for (int u = 0; u < UPT; ++u) {  // ... which now receives h_l of the source slots
      const int j = tid + NT * u;
#pragma unroll
      for (int c = 0; c < NC; ++c) {
        float hv[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int m = 4 * c + q;
          hv[q] = (m < Mp) ? pool_hidden_cta[(size_t)cc.lane[m0 + m] * lane_pool_h + (size_t)cc.src[m0 + m] * DH +
                                             (size_t)l * H + j]
                           : 0.f;
        }
        reinterpret_cast<float4*>(XA + (size_t)j * C::CP)[c] = make_float4(hv[0], hv[1], hv[2], hv[3]);
      }
    }
    named_bar_sync(1, NT);
    lin_pass<C, 3 * H, C::KT_HH, 1, C::RG, NC, false>(ring, full, empty, it, XA, acc, tid, lane);  // += W_hh_l h_l
    const float* bi = p.bih_up + (size_t)(l - 1) * 3 * H;
    const float* bhl = p.bhh_up + (size_t)(l - 1) * 3 * H;
    float hn_out[UPT][4 * NC];
#pragma unroll
    for (int u = 0; u < UPT; ++u) {
      const int j = tid + NT * u;
      const float bir = bi[j], biz = bi[H + j], bin = bi[2 * H + j];
      const float bhr = bhl[j], bhz = bhl[H + j], bhn = bhl[2 * H + j];
#pragma unroll
      for (int c = 0; c < NC; ++c) {
        const float4 hold = reinterpret_cast<const float4*>(XA + (size_t)j * C::CP)[c];
        const float ho[4] = {hold.x, hold.y, hold.z, hold.w};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int m = 4 * c + q;
          const float r = sigmoid_f32(__fadd_rn(__fadd_rn(acc[0 * UPT + u][m], bir), bhr));
          const float z = sigmoid_f32(__fadd_rn(__fadd_rn(acc[1 * UPT + u][m], biz), bhz));
          const float n = tanhf(__fadd_rn(__fadd_rn(ni[u][m], bin), __fmul_rn(r, __fadd_rn(acc[2 * UPT + u][m], bhn))));
          const float hnew = __fadd_rn(__fmul_rn(__fsub_rn(ho[q], n), z), n);
          hn_out[u][m] = (m < Mp) ? hnew : 0.f;
          if (m < Mp)
            pool_hidden_cta[(size_t)cc.lane[m0 + m] * lane_pool_h + (size_t)cc.dst[m0 + m] * DH + (size_t)l * H + j] = hnew;
        }
      }
    }
    named_bar_sync(1, NT);  // XB (this layer's input) is no longer read by anyone
#pragma unroll
    for (int u = 0; u < UPT; ++u)
#pragma unroll
      for (int c = 0; c < NC; ++c)
        reinterpret_cast<float4*>(XB + (size_t)(tid + NT * u) * C::CP)[c] =
            make_float4(hn_out[u][4 * c], hn_out[u][4 * c + 1], hn_out[u][4 * c + 2], hn_out[u][4 * c + 3]);
  }
  named_bar_sync(1, NT);
  if (tid == 0) { const long long now_ = clock64(); ph[2] += now_ - tmark; tmark = now_; }
  // ---------------- a = relu(W1 h' + b1)
  {
    float acc[C::R1][4 * NC];
    lin_pass<C, H, C::KT_1, C::KG1, C::R1, NC, true, XCL>(ring, full, empty, it, XB, acc, tid, lane, xrank, xsize);
    float out[UPT][4 * NC];
    ksplit_reduce<C, H, C::KG1, C::R1, UPT, NC>(acc, XA, out, tid);
    if constexpr (XCL) {
      static_assert(UPT * 4 * NC <= kXchVals, "cluster mode: W1 exchange in one round");
      float v[UPT * 4 * NC];
#pragma unroll
      for (int u = 0; u < UPT; ++u)
#pragma unroll
        for (int m = 0; m < 4 * NC; ++m) v[u * 4 * NC + m] = out[u][m];
      xch_allreduce<NT, UPT * 4 * NC>(*xc, v, tid);
#pragma unroll
      for (int u = 0; u < UPT; ++u)
#pragma unroll
        for (int m = 0; m < 4 * NC; ++m) out[u][m] = v[u * 4 * NC + m];
    }
#pragma unroll
    for (int u = 0; u < UPT; ++u)
#pragma unroll
      for (int c = 0; c < NC; ++c) {
        float4 v;
        v.x = fmaxf(__fadd_rn(out[u][4 * c + 0], b1r[u]), 0.f); v.y = fmaxf(__fadd_rn(out[u][4 * c + 1], b1r[u]), 0.f);
        v.z = fmaxf(__fadd_rn(out[u][4 * c + 2], b1r[u]), 0.f); v.w = fmaxf(__fadd_rn(out[u][4 * c + 3], b1r[u]), 0.f);
        reinterpret_cast<float4*>(XA + (size_t)(tid + NT * u) * C::CP)[c] = v;
      }
  }
  named_bar_sync(1, NT);
  if (tid == 0) { const long long now_ = clock64(); ph[3] += now_ - tmark; tmark = now_; }
  // ---------------- mean = W2 a + b2, then the running-mean update of the cluster
  {
    // old means of the source slots (issued before the pass to hide the L2 latency)
    float mu_old[4 * NC];
#pragma unroll
    for (int m = 0; m < 4 * NC; ++m)
      mu_old[m] = (m < Mp && tid < D)
                      ? pool_mean_cta[(size_t)cc.lane[m0 + m] * lane_pool_m + (size_t)cc.src[m0 + m] * D + tid]
                      : 0.f;
    float acc[C::R2][4 * NC];
    lin_pass<C, D, C::KT_2, C::KG2, C::R2, NC, true, XCL>(ring, full, empty, it, XA, acc, tid, lane, xrank, xsize);
    float out[1][4 * NC];
    ksplit_reduce<C, D, C::KG2, C::R2, 1, NC>(acc, XA, out, tid);
    if constexpr (XCL) xch_allreduce<NT, 4 * NC>(*xc, out[0], tid);
    if (tid < D) {
#pragma unroll
      for (int m = 0; m < 4 * NC; ++m) {
        if (m < Mp) {
          const float mval = __fadd_rn(out[0][m], b2r);
          const int n = cc.vis[m0 + m];  // visits BEFORE this one (uisrnn.py:425-429)
          // mean_set[c] = (mean_set[c] * (n - 1) + mean) / n   -- fp32, true division
          const float mu = (n == 0) ? mval
                                    : __fdiv_rn(__fadd_rn(__fmul_rn(mu_old[m], (float)(n - 1)), mval), (float)n);
          pool_mean_cta[(size_t)cc.lane[m0 + m] * lane_pool_m + (size_t)cc.dst[m0 + m] * D + tid] = mu;
        }
      }
    }
  }
}

// Picks the instantiation by NC = number of 4-column chunks in this pass.  DEEP (stacked GRU layers) is a
// template parameter of the kernels so that the depth-1 kernels carry none of that code or its registers.
template <class C, bool DEEP, bool XCL = false>
__device__ __forceinline__ void run_pass_any(const BeamParams& p, const float* ring, uint64_t* full, uint64_t* empty,
                                             unsigned& it, float* XA, float* XB, const ColCtx cc, int m0, int Mp,
                                             float* pool_mean_cta, float* pool_hidden_cta, const float (&bh)[C::RG],
                                             const float (&b1r)[C::UPT], float b2r, int tid, int lane, long long* ph,
                                             long long& tmark, XchCtx* xc = nullptr) {
  const int nc = (Mp + 3) / 4;
#define UIS_RP(NCV, DEEPV) \
  run_pass<C, NCV, DEEPV, XCL>(p, ring, full, empty, it, XA, XB, cc, m0, Mp, pool_mean_cta, pool_hidden_cta, bh, b1r, b2r, tid, lane, ph, tmark, xc)
  if (nc == 1) UIS_RP(1, DEEP); else if (nc == 2) UIS_RP(2, DEEP); else if (nc == 3 || C::CP < 16) UIS_RP(3, DEEP);
  else if (nc == 4 || C::CP < 20) { if constexpr (C::CP >= 16) UIS_RP(4, DEEP); }
  else { if constexpr (C::CP >= 20) UIS_RP(5, DEEP); }
#undef UIS_RP
}

// ---- stationary-weights pass (uis_beam_stat.cuh): columns [m0, m0 + Mp), Mp <= CP.  XA holds the source hidden states
// [H][CP] (gathered by the caller); CTA `q` of the group computes its rows of the three products from the weights
// resident in `sW` and publishes them through the group-shared slot pool / the L2 scratch; three group barriers.
template <int H, int D, int CP, int NT>
__device__ __forceinline__ void stat_pass(const BeamParams& p, const float* sW, float* XA, float* XB, const ColCtx cc, int m0,
                                          int Mp, float* pool_mean_g, float* pool_hidden_g, float* scratch_g, unsigned* bar,
                                          unsigned& epoch, int q, int tid, long long* ph, long long& tmark) {
  using S = StatCfg<H, D>;
  const size_t lane_pool_h = (size_t)p.P * H, lane_pool_m = (size_t)p.P * D;
  // ---------------- GRU: rows g * UG + u  ->  h' of units q * UG + u
  stat_dot<H, S::R0, CP, NT>(sW, S::LD, 0, XA, XB, Mp, tid);
  named_bar_sync(1, NT);
  if (tid < S::UG * CP) {
    const int m = tid % CP, u = tid / CP, j = q * S::UG + u;
    if (m < Mp) {
      const float ar = stat_sum<S::R0, CP, NT>(XB, 0 * S::UG + u, m);
      const float az = stat_sum<S::R0, CP, NT>(XB, 1 * S::UG + u, m);
      const float an = stat_sum<S::R0, CP, NT>(XB, 2 * S::UG + u, m);
      const float* gi = p.gi + (size_t)cc.girow[m0 + m] * 3 * H;
      const float r = sigmoid_f32(__fadd_rn(gi[j], __fadd_rn(ar, __ldg(p.bhh + j))));
      const float z = sigmoid_f32(__fadd_rn(gi[H + j], __fadd_rn(az, __ldg(p.bhh + H + j))));
      const float n = tanhf(__fadd_rn(gi[2 * H + j], __fmul_rn(r, __fadd_rn(an, __ldg(p.bhh + 2 * H + j)))));
      const float ho = XA[(size_t)j * CP + m];
      pool_hidden_g[(size_t)cc.lane[m0 + m] * lane_pool_h + (size_t)cc.dst[m0 + m] * H + j] =
          __fadd_rn(__fmul_rn(__fsub_rn(ho, n), z), n);   // h' = (h - n) * z + n
    }
  }
  stat_group_sync<NT>(bar, epoch, tid);
  if (tid == 0) { const long long now_ = clock64(); ph[2] += now_ - tmark; tmark = now_; }
  // ---------------- a = relu(W1 h' + b1): every CTA needs the whole h' columns (written by all CTAs of the group)
  // (column by column so that a warp reads 128 contiguous bytes of one new slot; columns >= Mp of XA are still the
  //  zeros the caller's gather of the source states put there)
  for (int i = tid; i < Mp * H; i += NT) {
    const int m = i / H, k = i % H;
    XA[(size_t)k * CP + m] = __ldcg(pool_hidden_g + (size_t)cc.lane[m0 + m] * lane_pool_h + (size_t)cc.dst[m0 + m] * H + k);
  }
  named_bar_sync(1, NT);
  stat_dot<H, S::R1, CP, NT>(sW, S::LD, S::R0, XA, XB, Mp, tid);
  named_bar_sync(1, NT);
  if (tid < S::R1 * CP) {
    const int m = tid % CP, u = tid / CP, j = q * S::R1 + u;
    if (m < Mp)
      scratch_g[(size_t)m * H + j] = fmaxf(__fadd_rn(stat_sum<S::R1, CP, NT>(XB, u, m), __ldg(p.b1 + j)), 0.f);
  }
  stat_group_sync<NT>(bar, epoch, tid);
  if (tid == 0) { const long long now_ = clock64(); ph[3] += now_ - tmark; tmark = now_; }
  // ---------------- mean = W2 a + b2, then the running-mean update of the cluster (uisrnn.py:425-429)
  for (int i = tid; i < Mp * H; i += NT) {
    const int m = i / H, k = i % H;
    XA[(size_t)k * CP + m] = __ldcg(scratch_g + (size_t)m * H + k);
  }
  named_bar_sync(1, NT);
  stat_dot<H, S::R2, CP, NT>(sW, S::LD, S::R0 + S::R1, XA, XB, Mp, tid);
  named_bar_sync(1, NT);
  if (tid < S::R2 * CP) {
    const int m = tid % CP, u = tid / CP, d = q * S::R2 + u;
    if (m < Mp) {
      const float mval = __fadd_rn(stat_sum<S::R2, CP, NT>(XB, u, m), __ldg(p.b2 + d));
      const int n = cc.vis[m0 + m];  // visits BEFORE this one
      const float mu_old = __ldcg(pool_mean_g + (size_t)cc.lane[m0 + m] * lane_pool_m + (size_t)cc.src[m0 + m] * D + d);
      const float mu = (n == 0) ? mval : __fdiv_rn(__fadd_rn(__fmul_rn(mu_old, (float)(n - 1)), mval), (float)n);
      pool_mean_g[(size_t)cc.lane[m0 + m] * lane_pool_m + (size_t)cc.dst[m0 + m] * D + d] = mu;
    }
  }
  stat_group_sync<NT>(bar, epoch, tid);  // the next step scores against the new means / gathers the new hidden states
}

// ---- tensor-core weight pass (consumer warps' side; uis_beam_tc.cuh has the TMA producer and the MMA tiles) -----
// Columns [m0, m0 + Mp), Mp <= N.  Warpgroup wg = warp / 4 multiplies rows 64 wg .. 64 wg + 63 of every 128-row tile;
// its accumulator layout gives a thread rows r0 and r0 + 8 and the columns 8 i + 2 (lane % 4) + {0, 1}.
// tstat: thread 0's pass counters ([0] box waits, [1] MMA waits, [2] B operand staging, [3] cycles inside passes).
template <int H, int D, int N, class Idle>
__device__ __forceinline__ void tc_run_pass(const BeamParams& p, const unsigned char* ring, unsigned char* bop,
                                            const TcBars& tb, unsigned& tbox, const ColCtx cc, int m0, int Mp,
                                            float* pool_mean_cta, float* pool_hidden_cta, float* scratch_cta, int tid,
                                            int lane, int warp, long long* ph, long long& tmark, long long* tstat,
                                            Idle idle_work) {
  using TC = TcCfg<H, D, N>;
  constexpr int NT = 256, NI = N / 8;
  // batch sizes of the GRU (KB columns) and running-mean (WB groups of 8 columns) epilogues: larger batches spill
  constexpr int KB = 2, WB = 3;
  // slot s of lane g in the CTA's pools (g * P + s is small: 32-bit index arithmetic, no 64-bit strides held)
  auto hslot = [&](int g, int s) { return pool_hidden_cta + (size_t)(g * p.P + s) * H; };
  auto mslot = [&](int g, int s) { return pool_mean_cta + (size_t)(g * p.P + s) * D; };
  const int wg = warp >> 2;
  const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const int cq = 2 * (lane & 3);
  long long* ts = (tid == 0) ? tstat : nullptr;
  const long long t_in = clock64();
  float acc[TC::NACC];
  auto stage_b = [&](auto src, float scale) {
    const long long w0 = clock64();
    tc_gather_b<H, N, NT>(bop, src, Mp, scale, tid);
    tc_publish_b<NT>();
    if (ts) ts[2] += clock64() - w0;
  };
  // gi rows of the pass's lanes (3H floats each; the columns of a lane are consecutive and share its row) to L2: gi
  // of the whole batch is far larger than L2, so the GRU epilogue would otherwise read them from HBM
  if (tid < Mp && (tid == 0 || cc.lane[m0 + tid] != cc.lane[m0 + tid - 1]))
    prefetch_l2_bulk(p.gi + (size_t)cc.girow[m0 + tid] * 3 * H, 3 * H * 4);
  // ---------------- B = h_src (fp16 hi / lo), then the GRU gates per 128-unit tile
  stage_b([&](int m) -> const float* {
    return hslot(cc.lane[m0 + m], cc.src[m0 + m]); }, p.tc_sh);
  if (tid == 0) { const long long now_ = clock64(); ph[1] += now_ - tmark; tmark = now_; }
  idle_work();  // the next step's Gaussian terms (their frame has landed by now)
  // (charged to the scoring phase: the TMA ring is already filled meanwhile, the MMAs wait for it)
  if (tid == 0) { const long long now_ = clock64(); ph[7] += now_ - tmark; tmark = now_; }
  // The r and z sums of a unit tile wait in this CTA's scratch (free until the W1 epilogue) while the n tile is
  // multiplied: held in registers next to its accumulator they would not fit the 168 registers of a thread.
  static_assert(H >= NT, "gate parking: 2 * (N / 2) * NT floats within the [N][H] scratch");
  float* park = scratch_cta + tid;
  for (int ut = 0; ut < TC::UT; ++ut) {
    // gate sums + b_hh: value 4 i + 2 h + e of a tile is row j0 + 8 h, so its bias is that of row j0 + 8 h
    const int j0 = ut * 128 + r0;
    {
      float v[TC::NV];
#pragma unroll
      for (int g = 0; g < 2; ++g) {  // r, z: parked
        tc_tile<TC>(acc, ring, bop, tb, tbox, wg, lane, ts);
        tc_fold<TC>(acc, v, p.tc_inv_hh);
        const float bh[2] = {__ldg(p.bhh + g * H + j0), __ldg(p.bhh + g * H + j0 + 8)};
#pragma unroll
        for (int q = 0; q < TC::NV; ++q) park[(g * TC::NV + q) * NT] = __fadd_rn(v[q], bh[(q >> 1) & 1]);
      }
    }
    tc_tile<TC>(acc, ring, bop, tb, tbox, wg, lane, ts);
    float an[TC::NV];
    tc_fold<TC>(acc, an, p.tc_inv_hh);
    {
      const float bh[2] = {__ldg(p.bhh + 2 * H + j0), __ldg(p.bhh + 2 * H + j0 + 8)};
#pragma unroll
      for (int q = 0; q < TC::NV; ++q) an[q] = __fadd_rn(an[q], bh[(q >> 1) & 1]);
    }
    // GRU cell, PyTorch gate order r,z,n:  h' = (h - n) * z + n, for this thread's rows j0 + 8 h of every column.
    // A batch of KB columns issues all its loads before its first store, so that their round trips to L2
    // overlap instead of queueing behind the stores.  Taking the loads ahead of earlier stores is safe: every store
    // goes to a new slot, which P3 took from the free bitmap, so it is never the source slot of a column of this
    // pass, and a slot is not modified once written; `park` is this thread's own; gi is read-only for the whole
    // kernel (non-coherent loads are fine), the slot pool is written by the kernel (coherent loads only).
#pragma unroll
    for (int k0 = 0; k0 < 2 * NI; k0 += KB) {  // k = 2 i + e: column 8 i + cq + e
      float gr[KB][2], gz[KB][2], gn[KB][2], pr[KB][2], pz[KB][2], ho[KB][2];  // [k - k0][h]
#pragma unroll
      for (int b = 0; b < KB; ++b) {
        const int i = (k0 + b) >> 1, e = (k0 + b) & 1, m = 8 * i + cq + e;
        if (m < Mp) {
          const float* gi = p.gi + (size_t)cc.girow[m0 + m] * 3 * H + j0;
          const float* hs = hslot(cc.lane[m0 + m], cc.src[m0 + m]) + j0;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int v = 4 * i + 2 * h + e;
            gr[b][h] = __ldg(gi + 8 * h); gz[b][h] = __ldg(gi + H + 8 * h); gn[b][h] = __ldg(gi + 2 * H + 8 * h);
            pr[b][h] = park[v * NT]; pz[b][h] = park[(TC::NV + v) * NT];
            ho[b][h] = hs[8 * h];
          }
        }
      }
#pragma unroll
      for (int b = 0; b < KB; ++b) {
        const int i = (k0 + b) >> 1, e = (k0 + b) & 1, m = 8 * i + cq + e;
        if (m < Mp) {
          float* hd = hslot(cc.lane[m0 + m], cc.dst[m0 + m]) + j0;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int v = 4 * i + 2 * h + e;
            const float rg = sigmoid_f32(__fadd_rn(gr[b][h], pr[b][h]));
            const float zg = sigmoid_f32(__fadd_rn(gz[b][h], pz[b][h]));
            const float ng = tanhf(__fadd_rn(gn[b][h], __fmul_rn(rg, an[v])));
            hd[8 * h] = __fadd_rn(__fmul_rn(__fsub_rn(ho[b][h], ng), zg), ng);
          }
        }
      }
    }
  }
  named_bar_sync(1, NT);  // h' of every column is in the slot pool (global memory, CTA-scope ordering)
  if (tid == 0) { const long long now_ = clock64(); ph[2] += now_ - tmark; tmark = now_; }
  // ---------------- B = h', a = relu(W1 h' + b1) -> scratch
  stage_b([&](int m) -> const float* {
    return hslot(cc.lane[m0 + m], cc.dst[m0 + m]); }, p.tc_sh);
  for (int mt = 0; mt < TC::T2; ++mt) {
    float v1[TC::NV];
    tc_tile<TC>(acc, ring, bop, tb, tbox, wg, lane, ts);
    tc_fold<TC>(acc, v1, p.tc_inv_1);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int j = mt * 128 + r0 + 8 * h;
      const float b1j = __ldg(p.b1 + j);
#pragma unroll
      for (int i = 0; i < NI; ++i)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int m = 8 * i + cq + e;
          if (m < Mp) scratch_cta[(size_t)m * H + j] = fmaxf(__fadd_rn(v1[4 * i + 2 * h + e], b1j), 0.f);
        }
    }
  }
  named_bar_sync(1, NT);
  if (tid == 0) { const long long now_ = clock64(); ph[3] += now_ - tmark; tmark = now_; }
  // ---------------- B = a, mean = W2 a + b2, then the running-mean update of the cluster
  stage_b([&](int m) -> const float* { return scratch_cta + (size_t)m * H; }, p.tc_sa);
  for (int mt = 0; mt < TC::T3; ++mt) {
    float v2[TC::NV];
    tc_tile<TC>(acc, ring, bop, tb, tbox, wg, lane, ts);
    tc_fold<TC>(acc, v2, p.tc_inv_2);
    // the old means of a batch of WB column groups are loaded before the first new mean is stored (a new slot is never
    // the source slot of a column of this pass, see the GRU epilogue)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int d = mt * 128 + r0 + 8 * h;
      const float b2d = __ldg(p.b2 + d);
#pragma unroll
      for (int i0 = 0; i0 < NI; i0 += WB) {
        float mu_old[WB][2];
#pragma unroll
        for (int b = 0; b < WB; ++b)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int m = 8 * (i0 + b) + cq + e;
            if (m < Mp) mu_old[b][e] = mslot(cc.lane[m0 + m], cc.src[m0 + m])[d];
          }
#pragma unroll
        for (int b = 0; b < WB; ++b)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int m = 8 * (i0 + b) + cq + e;
            if (m < Mp) {
              const float mval = __fadd_rn(v2[4 * (i0 + b) + 2 * h + e], b2d);
              const int n = cc.vis[m0 + m];  // visits BEFORE this one
              // mean_set[c] = (mean_set[c] * (n - 1) + mean) / n   -- fp32, true division
              const float mu = (n == 0) ? mval : __fdiv_rn(__fadd_rn(__fmul_rn(mu_old[b][e], (float)(n - 1)), mval), (float)n);
              mslot(cc.lane[m0 + m], cc.dst[m0 + m])[d] = mu;
            }
          }
      }
    }
  }
  if (ts) ts[3] += clock64() - t_in;
}

// ------------------------------------------------------------------ the kernel
// XCL = cluster (latency) mode: the kernel is launched with thread-block clusters of 2/4/8 CTAs; the CTAs of a
// cluster run the SAME utterances in lock step (all selection phases replicated, bit-identical), and split every
// weight matrix by k-tiles, exchanging partial sums through distributed shared memory (xch_allreduce).
// TCN > 0 = tensor-core pass (uis_beam_tc.cuh): the three matrix products of the step run as wgmma MMAs over
// TCN columns per pass, issued by the two consumer warpgroups; warp NW drives the tensor-map TMA.
// XM = 2: stationary-weights mode (uis_beam_stat.cuh): groups of 32 CTAs, one utterance stream per group, weights
// resident in shared memory, products split by rows, group barriers in global memory (cooperative launch).
template <int H, int D, bool DEEP, int XM = 0, int TCN = 0>
__global__ void __launch_bounds__(Cfg<H, D>::BLOCK, 1) uis_beam_kernel(const __grid_constant__ BeamParams p) {
  constexpr bool XCL = XM == 1, STAT = XM == 2;
  using C = Cfg<H, D, (XCL || STAT) ? kCPCluster : BeamCP<H>::value>;
  constexpr int NT = C::NT, NW = C::NW, UPT = C::UPT;
  constexpr bool TC = TCN > 0;
  static_assert(!TC || (!DEEP && !XCL && !STAT && NT == 256 && C::REBALANCE), "tensor-core pass: depth 1, one CTA per lane group");
  static_assert(!STAT || (!DEEP && NT == 256), "stationary-weights mode: depth 1, 256 consumer threads");
  using TCC = TcCfg<TC ? H : 512, TC ? D : 256, TC ? TCN : 48>;  // (a valid placeholder for the FFMA kernels)
  extern __shared__ __align__(128) unsigned char smem_raw[];
  // the swizzled TMA boxes / MMA operands of the tensor-core pass need 1024-byte alignment
  unsigned char* smem = TC ? reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023)
                           : smem_raw;
  const int B = p.B, Kcap = p.Kcap, G = p.G;
  const SmemLayout L_ = make_layout<H, D, C::CP, XCL, TCN, STAT>(B, Kcap, G);
  const SmemLayout& L = TC ? p.tc_layout : L_;  // tensor-core engine: read from the parameter bank, no registers
  if constexpr (TC)
    if (p.tc_layout.total == 0) __trap();  // a launcher that did not fill tc_layout (launch_beam_tc does)
  const int sq = STAT ? (int)(blockIdx.x % kStatGroup) : 0, sgroup = STAT ? (int)(blockIdx.x / kStatGroup) : 0;
  float* ring = reinterpret_cast<float*>(smem + L.ring);
  float* XA = reinterpret_cast<float*>(smem + L.xa);
  float* XB = reinterpret_cast<float*>(smem + L.xb);
  float* wv = reinterpret_cast<float*>(smem + L.wv);
  int* colarr = reinterpret_cast<int*>(smem + L.cols);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + L.bars);
  uint64_t* empty = full + (TC ? TCC::STAGES : kStages);
  volatile int* misc = reinterpret_cast<volatile int*>(smem + L.misc);
  TcBars tb{full, empty};

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  if (tid == 0) {
    if constexpr (TC) {
      for (int s = 0; s < TCC::STAGES; ++s) {
        mbar_init(&tb.full[s], 1);
        mbar_init(&tb.empty[s], NW);
      }
    } else {
      for (int s = 0; s < kStages; ++s) {
        mbar_init(&full[s], 1);
        mbar_init(&empty[s], NW);
      }
    }
    for (int i = 0; i < 16; ++i) misc[i] = 0;
    if constexpr (TC)
      for (int i = 16; i < 20; ++i) reinterpret_cast<long long*>(smem + L.phase)[i] = 0;
    if constexpr (XCL) {
      uint64_t* xbar = reinterpret_cast<uint64_t*>(smem + L.xbar);
      mbar_init(&xbar[0], cluster_nctarank() - 1);
      mbar_init(&xbar[1], cluster_nctarank() - 1);
      misc[MI_QNEXT] = (int)cluster_id_x();  // utterances are dealt to the clusters round-robin (no atomic queue)
    }
    if constexpr (STAT) misc[MI_QNEXT] = sgroup;  // ... and to the groups of the stationary-weights mode
    fence_mbar_init();
  }
  __syncthreads();
  if constexpr (XCL) cluster_sync_all();  // every peer's exchange barriers exist before anyone arrives on them

  if (warp >= NW) {  // ---------------- producer warp (+ idle warps of its warpgroup)
    if constexpr (STAT) return;  // nothing streams: the weights are resident
    if constexpr (TC) asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    else if constexpr (C::REBALANCE) asm volatile("setmaxnreg.dec.sync.aligned.u32 24;");
    if constexpr (TC) {
      if (warp == NW) tc_producer_loop<TCC, H>(&p.tc_wmap, reinterpret_cast<unsigned char*>(ring), tb, &misc[MI_DONE]);
    } else {
      if (warp == NW && lane == 0) producer_loop<C, XCL>(p, ring, full, empty, misc);
    }
    return;
  }
  if constexpr (TC) asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");  // 8 x 32 x 232 + 4 x 32 x 40 <= 64 K registers
  else if constexpr (C::REBALANCE && !STAT) asm volatile("setmaxnreg.inc.sync.aligned.u32 240;");

  // ---------------- consumer threads (tid < NT); they synchronise on named barrier 1
  auto lane_base = [&](int g) -> unsigned char* { return smem + L.lanes + (size_t)g * L.lane_stride; };
  auto LSp = [&](int g) -> volatile int* { return reinterpret_cast<volatile int*>(lane_base(g) + L.l_ls); };
  const int DH = p.depth * H;
  const size_t pool_m_stride = (size_t)p.P * D, pool_h_stride = (size_t)p.P * DH;
  // (stationary-weights mode: the CTAs of a group share ONE slot pool -- every CTA writes its rows of the new slots)
  float* pool_mean_cta = p.pool_mean + (size_t)(STAT ? sgroup : blockIdx.x) * G * pool_m_stride;
  float* pool_hidden_cta = p.pool_hidden + (size_t)(STAT ? sgroup : blockIdx.x) * G * pool_h_stride;
  unsigned* bp_cta = p.bp + (size_t)blockIdx.x * G * p.maxN * B;
  const unsigned PW = (unsigned)(p.P + 31) / 32;
  const float INF = __int_as_float(0x7f800000);
  const int bbits = B > 32 ? 7 : 5;  // bits of the hypothesis index inside a candidate record (phase P1)

  float bh[C::RG], b1r[UPT];
#pragma unroll
  for (int i = 0; i < C::RG; ++i) bh[i] = TC ? 0.f : p.bhh[(i / UPT) * H + tid + NT * (i % UPT)];
#pragma unroll
  for (int u = 0; u < UPT; ++u) b1r[u] = TC ? 0.f : p.b1[tid + NT * u];
  const float b2r = (tid < D && !TC) ? p.b2[tid] : 0.f;
  unsigned tc_boxes = 0;  // tensor-core pass: ring boxes consumed so far (identical in every consumer thread)
  float* tc_scratch_cta = TC ? p.tc_scratch + (size_t)blockIdx.x * (TC ? TCN : 1) * H : nullptr;
  if (tid < D) wv[tid] = p.wvec[tid];
  unsigned stat_epoch = 0;
  if constexpr (STAT) stat_load_weights<H, D, NT>(ring, p.whh_t, p.w1_t, p.w2_t, sq, tid);
  for (int g = 0; g < G; ++g) {
    if (tid < D) pool_mean_cta[g * pool_m_stride + (size_t)kInitSlot * D + tid] = p.mean0[tid];
    for (int q = tid; q < DH; q += NT) pool_hidden_cta[g * pool_h_stride + (size_t)kInitSlot * DH + q] = p.hidden0[q];
  }

  int* collane = colarr; int* colsrc = colarr + G * B; int* colnew = colarr + 2 * G * B;
  int* colvis = colarr + 3 * G * B;
  long long* colrow = reinterpret_cast<long long*>(colarr + 4 * G * B);
  const ColCtx cc{collane, colsrc, colnew, colvis, colrow};
  XchCtx xc{reinterpret_cast<float*>(smem + L.xch), reinterpret_cast<uint64_t*>(smem + L.xbar),
            XCL ? cluster_ctarank() : 0u, XCL ? cluster_nctarank() : 1u, 0u};
  const int xsize = (int)xc.size;
  // Debug taps: the CTAs of a cluster / group decode the same utterance in lock step, and one of them writes the taps
  const bool tap_leader = (!XCL || xc.rank == 0) && (!STAT || sq == 0);

  unsigned it = 0;  // weight-ring tile counter (identical in every consumer thread)
  // Statistics are thread 0's alone and live in shared memory: as locals they would hold ~30 registers in
  // every thread across the whole kernel.  ph[0..9]: per-phase cycle counters, ph[10]: phase mark,
  // ph[11..15]: columns, passes, candidates, steps, max K.
  long long* ph = reinterpret_cast<long long*>(smem + L.phase);
  if (tid == 0) {
    for (int i = 0; i < 16; ++i) ph[i] = 0;
    ph[10] = clock64();
  }
  // (ph[16..19], the tensor-core pass counters, are zeroed by thread 0 before the first __syncthreads)
  long long& tmark = ph[10];
  long long& st_cols = ph[11]; long long& st_pass = ph[12]; long long& st_cand = ph[13]; long long& st_steps = ph[14];
  long long& st_maxk = ph[15];
#define UIS_PHASE(i)                         \
  do {                                       \
    if (tid == 0) {                          \
      const long long now_ = clock64();      \
      ph[i] += now_ - tmark;                 \
      tmark = now_;                          \
    }                                        \
  } while (0)

  // Pull the next non-empty utterance for lane g (one thread).
  auto lane_fetch = [&](int g) {
    volatile int* ls = LSp(g);
    for (;;) {
      int uidx;
      if constexpr (XCL) {  // one lane per cluster; every CTA of the cluster draws the same sequence
        uidx = misc[MI_QNEXT];
        misc[MI_QNEXT] = uidx + (int)cluster_nclusters_x();
      } else if constexpr (STAT) {
        uidx = misc[MI_QNEXT];
        misc[MI_QNEXT] = uidx + (int)(gridDim.x / kStatGroup);
      } else {
        uidx = atomicAdd(p.queue, 1);
      }
      if (uidx >= p.U) { ls[LS_ACTIVE] = 0; ls[LS_FRESH] = 0; return; }
      const int u = p.order[uidx], utt = u % p.n_utt;  // u: the job
      const long long row0 = p.row_off[utt];
      const int N = (int)(p.row_off[utt + 1] - row0);
      if (N == 0) {
        p.status[u] = 0;
        if (p.spk_out) p.spk_out[u] = 0;
        if (p.nbest_count) p.nbest_count[u] = 0;
        for (int j = 0; j < p.n_best; ++j) nbest_store(p, u, j, -1, nullptr, nullptr);
        if (p.dbg_final_scores && tap_leader) {
          for (int b = 0; b < B; ++b) p.dbg_final_scores[(size_t)u * B + b] = INF;
          if (p.dbg_final_k) p.dbg_final_k[u] = 0;
        }
        continue;
      }
      ls[LS_U] = u; ls[LS_N] = N; ls[LS_TN] = p.T * N; ls[LS_T] = 0; ls[LS_NB] = 1; ls[LS_GEN] = 0;
      ls[LS_ACTIVE] = 1; ls[LS_FAILED] = 0; ls[LS_TRACED] = (u == p.trace_utt) && tap_leader; ls[LS_ERR] = 0;
      ls[LS_ROW0_LO] = (int)(row0 & 0xffffffffll); ls[LS_ROW0_HI] = (int)(row0 >> 32);
      ls[LS_DBGROWS_LO] = 0; ls[LS_DBGROWS_HI] = 0; ls[LS_FRESH] = 1;
      ls[LS_KHI] = spk_max(p, utt); ls[LS_KLO] = spk_min(p, utt);
      for (unsigned w = 0; w < PW; ++w) reinterpret_cast<unsigned*>(lane_base(g) + L.l_scored)[w] = 0;
      int* meta = reinterpret_cast<int*>(lane_base(g) + L.l_meta);  // [gen][field][B]: K,last,tot,nl
      meta[0] = 0; meta[B] = -1; meta[2 * B] = 0; reinterpret_cast<float*>(meta)[3 * B] = 0.f;
      if (u == p.trace_utt && tap_leader && p.dbg_off) p.dbg_off[0] = 0;
      return;
    }
  };
  // Lane teams.  The lanes are independent outside the weight pass, so the consumer warps split into G teams of
  // TW = NW / G warps and team t runs every selection phase of lane t (P0-P4, the Gaussian terms of its slots, P6) on
  // its own: a one-warp team synchronises with __syncwarp, a larger one on named barrier 2 + t (barrier 1 is the
  // consumers').  Warps past G * TW own no lane.  The lanes meet only around the pass: after every team has published
  // its lane's column count M, after the CTA column list is written, and at the pass's own barriers.  (team, ttid,
  // twarp) are recomputed from `warp` and p.G where needed, so they hold no registers across the pass.
  if (G > NW) __trap();  // the launcher runs at most one lane per consumer warp
  auto team_of = [&]() { return warp / (NW / G); };
  auto team_sync = [&]() {
    const int TW = NW / G;
    if (TW == 1) __syncwarp();
    else named_bar_sync(2 + warp / TW, TW * 32);
  };

  // Team threads of lane g: start the cp.async of frame `t` of lane g into buffer (t & 1).  The team waits for its
  // own copies (cp.async completion is per thread).
  auto lane_prefetch = [&](int g, int t, int ttid, int TT) {
    volatile int* ls = LSp(g);
    const long long row0 = ((long long)ls[LS_ROW0_HI] << 32) | (unsigned)ls[LS_ROW0_LO];
    const long long r = row0 + (t % ls[LS_N]);
    float* xts = reinterpret_cast<float*>(lane_base(g) + L.l_xt) + (t & 1) * D;
    for (int q = ttid; q < D / 4; q += TT) cp_async16(xts + q * 4, p.x + (size_t)r * D + q * 4);
  };

  // Gaussian terms of lane g's slots, by the team of lane g (it synchronises on the team barrier).
  //   next == false (phase P1): slots of `used` without a bit in `scored`, against the current frame x_t;
  //   next == true  (tensor-core engine, while the first tiles of the weight pass are multiplied): every slot the
  //   caller marked in `scored` (the next generation's live slots, new slots excluded), against x_{t+1}.
  // weighted_mse_loss for one row (loss_func.py:33-41): sum_d fl(fl(diff^2) * w_d), divided by the count of rows
  // whose first squared difference is non-zero (0 -> inf / nan); stored per slot in pool_mse.
  float* pool_mse_cta = p.pool_mse + (size_t)blockIdx.x * G * p.P;
  constexpr int kSlotList = 64;  // slots per listing round and lane
  auto score_lane_slots = [&](int g, bool next, int ttid, int twarp, int TW) {
    unsigned* used = reinterpret_cast<unsigned*>(lane_base(g) + L.l_used);
    unsigned* scored = reinterpret_cast<unsigned*>(lane_base(g) + L.l_scored);
    unsigned* slist = reinterpret_cast<unsigned*>(smem + L.slist) + kSlotList * g;
    volatile int* ls = LSp(g);
    const float* xs = reinterpret_cast<const float*>(lane_base(g) + L.l_xt) + ((ls[LS_T] + (next ? 1 : 0)) & 1) * D;
    const float* mu_g = pool_mean_cta + g * pool_m_stride;
    float* mse_g = pool_mse_cta + (size_t)g * p.P;
    for (;;) {
      if (twarp == 0) {  // the team's first warp lists the slots: a prefix over the bitmap words, 32 words per round
        int ntot = 0;
        for (int w0 = 0; w0 < (int)PW; w0 += 32) {
          const int w = w0 + lane;
          unsigned bits = 0;
          if (w < (int)PW) bits = next ? (scored[w] & ~used[w]) : (used[w] & ~scored[w]);  // (next: `used` = listed)
          const int n = __popc(bits);
          int incl = n;
#pragma unroll
          for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += v;
          }
          int pos = ntot + incl - n;
          unsigned done = 0;
          while (bits && pos < kSlotList) {
            const int bit = __ffs(bits) - 1;
            bits &= bits - 1;
            done |= 1u << bit;
            slist[pos++] = (unsigned)(w * 32 + bit);
          }
          if (done) { if (next) used[w] |= done; else scored[w] |= done; }
          ntot += __shfl_sync(0xffffffffu, incl, 31);
        }
        if (lane == 0) ls[LS_NLIST] = ntot;
      }
      team_sync();
      const int ntot = ls[LS_NLIST], nlist = min(ntot, kSlotList);
      // one warp per slot; each warp takes kBatch slots per trip and issues all their slot-pool loads (L2) before
      // reducing any of them, so the L2 round trips overlap instead of serialising
      constexpr int kBatch = 4;
      for (int f0 = twarp * kBatch; f0 < nlist; f0 += TW * kBatch) {
        int cslot[kBatch];
        float4 m4[kBatch][(D + 127) / 128];
#pragma unroll
        for (int q = 0; q < kBatch; ++q) {
          const int f = f0 + q;
          cslot[q] = -1;
          if (f < nlist) {
            cslot[q] = (int)slist[f];
            const float* mu = mu_g + (size_t)cslot[q] * D;
#pragma unroll
            for (int i = 0; i < (D + 127) / 128; ++i)
              if (lane * 4 + i * 128 < D)
                m4[q][i] = STAT ? __ldcg(reinterpret_cast<const float4*>(mu + lane * 4 + i * 128))  // written by other CTAs
                                : *reinterpret_cast<const float4*>(mu + lane * 4 + i * 128);
          }
        }
        bool live[kBatch];
#pragma unroll
        for (int q = 0; q < kBatch; ++q) live[q] = cslot[q] >= 0;
        const float my_term = gauss_rows<D, kBatch>(m4, live, xs, wv, lane);
        // lane q stores slot q
        int my_slot = cslot[0];
#pragma unroll
        for (int q = 1; q < kBatch; ++q)
          if (lane == q) my_slot = cslot[q];
        if (lane < kBatch && my_slot >= 0) mse_g[my_slot] = my_term;
      }
      team_sync();  // the terms are visible to the whole team (ordering of global memory among the team's threads)
      if (ntot <= kSlotList) break;  // (more slots than the list holds: another round over the unlisted ones)
    }
  };

  if (team_of() < G) {
    const int g = team_of(), TT = (NW / G) * 32, ttid = tid - g * TT;
    if (ttid == 0) lane_fetch(g);
    team_sync();
    if (LSp(g)[LS_ACTIVE]) lane_prefetch(g, 0, ttid, TT);
    cp_async_commit();
  }
  named_bar_sync(1, NT);  // slot 0 of every lane's pool and the MSE weights are written

  for (;;) {
    if (team_of() < G) {
      const int g = team_of(), TW = NW / G, TT = TW * 32, ttid = tid - g * TT, twarp = warp - g * TW;
      volatile int* ls = LSp(g);
      unsigned char* lb = lane_base(g);
      const bool active = ls[LS_ACTIVE] != 0;
      const int gen = ls[LS_GEN], t = ls[LS_T];
      const int* mK = reinterpret_cast<const int*>(lb + L.l_meta) + gen * 4 * B;
      const int* mLast = mK + B; const int* mTot = mK + 2 * B;
      const float* mNl = reinterpret_cast<const float*>(mK + 3 * B);
      int* candoff = reinterpret_cast<int*>(lb + L.l_candoff);
      const TabEntry* tab = reinterpret_cast<const TabEntry*>(lb + L.l_tabs) + (size_t)gen * B * Kcap;
      unsigned* used = reinterpret_cast<unsigned*>(lb + L.l_used);
      unsigned* scored = reinterpret_cast<unsigned*>(lb + L.l_scored);
      int* wins = reinterpret_cast<int*>(lb + L.l_wins);
      int* wcol = reinterpret_cast<int*>(lb + L.l_wcol);
      int* lcolsrc = reinterpret_cast<int*>(lb + L.l_lcol);
      int* lcolnew = lcolsrc + B;

      // ---- P0: candidate offsets of the lane; land x_t
      if (ttid == 0) {
        ls[LS_M] = 0; ls[LS_NWIN] = 0; ls[LS_NE] = 0;
        if (active) {
          int off = 0, kmax = 0;
          const int nb = ls[LS_NB], khi = ls[LS_KHI];
          // a hypothesis at max_speakers clusters has no new-cluster candidate (its score would be +inf); the flat
          // tie-break index below keeps the unbounded (kmax + 1) stride
          for (int b = 0; b < nb; ++b) { candoff[b] = off; off += mK[b] + (mK[b] < khi ? 1 : 0); kmax = max(kmax, mK[b]); }
          candoff[nb] = off;
          ls[LS_NFINITE] = 0; ls[LS_KMAX] = kmax; ls[LS_NE] = off;
        }
      }
      for (unsigned w = ttid; w < PW; w += TT) {
        used[w] = (w == 0) ? 1u : 0u;  // slot 0 = INIT, always live
        if (!TC) scored[w] = 0;        // (tensor-core engine: set by the pre-scoring of the previous step's pass)
      }
      cp_async_wait_all();
      team_sync();
      UIS_PHASE(6);
      if (active && t + 1 < ls[LS_TN]) lane_prefetch(g, t + 1, ttid, TT);  // the lane's next frame
      cp_async_commit();

      if (active) {
        // ---- P1: score every candidate (b, c <= K_b) of the lane  (uisrnn.py:409-420 existing cluster, :434-446 new
        //          cluster).  The Gaussian term depends only on (slot, x_t) -- hypotheses share most of their
        //          clusters' states -- so it is evaluated once per LIVE SLOT (one warp each), not once per candidate;
        //          slots whose term against x_t was already computed during the previous weight pass (tensor-core
        //          engine: the consumer warps idle while the first tiles are multiplied) are skipped.
        const int ne = ls[LS_NE], kmax = ls[LS_KMAX];
        double* pens = reinterpret_cast<double*>(lb + L.l_keys);
        unsigned long long* keys = reinterpret_cast<unsigned long long*>(lb + L.l_keys);
        unsigned* svals = reinterpret_cast<unsigned*>(lb + L.l_svals);
        // P1a: one thread per candidate resolves (hypothesis, cluster) -> slot, marks the slot live, and evaluates the
        // transition / ddCRP term in fp64 from the host-built log tables (the np.log values of uisrnn.py:415-420,
        // 444-446).  Parked in keys[] / svals[].  A thread's candidates grow, so its hypothesis index only moves on.
        const JobLogs lg = job_logs(p, ls[LS_U] / p.n_utt);
        int b = 0;
        for (int e = ttid; e < ne; e += TT) {
          while (candoff[b + 1] <= e) ++b;
          const int c = e - candoff[b];
          int slot = kInitSlot;
          double pen;
          if (c < mK[b]) {
            const TabEntry en = tab[(size_t)b * Kcap + c];
            slot = en.slot;
            atomicOr(used + (slot >> 5), 1u << (slot & 31));
            pen = (c == mLast[b]) ? lg.log_1mp0 : (lg.log_p0 + __ldg(p.logn + en.blocks)) - __ldg(lg.logtot + mTot[b]);
          } else {
            pen = (lg.log_p0 + lg.log_alpha) - __ldg(lg.logtot + mTot[b]);
          }
          pens[e] = pen;
          // slot (16 bits) | hypothesis (5 bits, or 7 when beam_size > 32: the host then caps kcap at 511) | cluster
          svals[e] = (unsigned)slot | ((unsigned)b << 16) | ((unsigned)c << (16 + bbits));
        }
        team_sync();
        // P1s: the live slots that still lack their term against x_t
        score_lane_slots(g, /*against the next frame=*/false, ttid, twarp, TW);
        // P1c: one thread per candidate: loss = fl32(f64(mse) - log terms); neg_likelihood accumulates in fp32
        //      (uisrnn.py:452); ranking key; the finite scores are counted per warp
        const float* mse_g = pool_mse_cta + (size_t)g * p.P;
        int nfin = 0;
        for (int e0 = 0; e0 < ne; e0 += TT) {
          const int e = e0 + ttid;
          bool finite = false;
          if (e < ne) {
            const unsigned info = svals[e];
            const int bb = (int)((info >> 16) & ((1u << bbits) - 1u)), c = (int)(info >> (16 + bbits));
            const float mse = mse_g[info & 0xffffu];
            const float loss = __double2float_rn((double)mse - pens[e]);
            const float S = __fadd_rn(mNl[bb], loss);
            reinterpret_cast<float*>(svals)[e] = S;
            const unsigned flat = (unsigned)(bb * (kmax + 1) + c);
            keys[e] = ((unsigned long long)float_order_key(S) << 32) | flat;
            finite = S < INF;
          }
          nfin += __popc(__ballot_sync(0xffffffffu, finite));
        }
        if (lane == 0 && nfin) atomicAdd((int*)&ls[LS_NFINITE], nfin);
        team_sync();
        UIS_PHASE(7);

        // ---- P2: rank by counting; the best min(#finite, B) become the new hypotheses (:546-552)
        const int nwin = min((int)ls[LS_NFINITE], B);
        b = 0;
        for (int e = ttid; e < ne; e += TT) {
          const unsigned long long k = keys[e];
          int rank = 0;
          for (int q = 0; q < ne; ++q) rank += (keys[q] < k) ? 1 : 0;
          if (rank < nwin) {
            while (candoff[b + 1] <= e) ++b;
            wins[rank] = b;
            wins[B + rank] = e - candoff[b];
            reinterpret_cast<float*>(wins)[2 * B + rank] = reinterpret_cast<const float*>(svals)[e];
          }
        }
        if (ttid == 0) ls[LS_NWIN] = nwin;
        team_sync();
        UIS_PHASE(8);

        // ---- P3: the team's first warp assigns the lane's GRU columns (distinct source slots) and allocates new
        //          slots; every warp of the team copies its share of the parents' tables into the next generation
        if (nwin > 0) {
          if (twarp == 0) {
            int M = 0;
            if (nwin <= 32) {  // one winner per lane (beam_size <= 32, or fewer finite candidates)
              const int r = lane;
              int src = -1;
              if (r < nwin) {
                const int wb = wins[r], c = wins[B + r];
                src = (c < mK[wb]) ? tab[(size_t)wb * Kcap + c].slot : kInitSlot;
              }
              int first = r;
              for (int q = 0; q < nwin; ++q) {
                const int sq_ = __shfl_sync(0xffffffffu, src, q);
                if (q < first && sq_ == src) first = q;
              }
              const bool isfirst = (r < nwin) && (first == r);
              const unsigned fm = __ballot_sync(0xffffffffu, isfirst);
              const int mycol = __popc(fm & ((1u << lane) - 1));
              M = __popc(fm);
              const int c_of_first = __shfl_sync(0xffffffffu, mycol, first);
              if (r < nwin) wcol[r] = c_of_first;
              if (isfirst) lcolsrc[mycol] = src;
            } else {
              // beam_size > 32: the winners are walked in chunks of 32; their source slots are parked in lcolnew
              // (rewritten by the slot allocation below) so that every winner can look for an earlier winner with the
              // same source
              for (int r = lane; r < nwin; r += 32) {
                const int wb = wins[r], c = wins[B + r];
                lcolnew[r] = (c < mK[wb]) ? tab[(size_t)wb * Kcap + c].slot : kInitSlot;
              }
              __syncwarp();
              for (int r0 = 0; r0 < nwin; r0 += 32) {  // columns are numbered in winner order, as in the one-chunk case
                const int r = r0 + lane;
                int first = r, src = -1;
                if (r < nwin) {
                  src = lcolnew[r];
                  for (int q = 0; q < r; ++q)
                    if (lcolnew[q] == src) { first = q; break; }
                }
                const bool isfirst = (r < nwin) && (first == r);
                const unsigned fm = __ballot_sync(0xffffffffu, isfirst);
                if (isfirst) {
                  const int mycol = M + __popc(fm & ((1u << lane) - 1));
                  wcol[r] = mycol;
                  lcolsrc[mycol] = src;
                }
                M += __popc(fm);
                __syncwarp();
                if (r < nwin && !isfirst) wcol[r] = wcol[first];  // `first` is an earlier winner: its column is already there
                __syncwarp();
              }
              __syncwarp();
            }
            // allocate M free slots from the bitmap (any free slot will do)
            int cnt = 0;
            for (unsigned w = lane; w < PW; w += 32) {
              unsigned fr = ~used[w];
              if (w == PW - 1 && (p.P & 31)) fr &= (1u << (p.P & 31)) - 1;
              cnt += __popc(fr);
            }
            int incl = cnt;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
              const int v = __shfl_up_sync(0xffffffffu, incl, o);
              if (lane >= o) incl += v;
            }
            int idx = incl - cnt;
            for (unsigned w = lane; w < PW && idx < M; w += 32) {
              unsigned fr = ~used[w];
              if (w == PW - 1 && (p.P & 31)) fr &= (1u << (p.P & 31)) - 1;
              while (fr && idx < M) {
                const int bit = __ffs(fr) - 1;
                fr &= fr - 1;
                lcolnew[idx++] = (int)(w * 32 + bit);
              }
            }
            if (lane == 0) ls[LS_M] = M;
          }
          // parents' tables -> next generation: winner r goes to warp r % TW of the team
          TabEntry* ntab = reinterpret_cast<TabEntry*>(lb + L.l_tabs) + (size_t)(gen ^ 1) * B * Kcap;
          for (int r = twarp; r < nwin; r += TW) {
            const int wb = wins[r];
            const int Kb = mK[wb];
            for (int c = lane; c < Kb; c += 32) ntab[(size_t)r * Kcap + c] = tab[(size_t)wb * Kcap + c];
          }
          team_sync();
          UIS_PHASE(9);

          // ---- P4: patch the one changed table entry per child; back-pointers; hypothesis meta.  The visit count of
          //          each lane-local column goes to lvis (the ranking keys are dead from here on) until the CTA
          //          column list is built.
          int* meta = reinterpret_cast<int*>(lb + L.l_meta);
          int* nK = meta + (gen ^ 1) * 4 * B; int* nLast = nK + B; int* nTot = nK + 2 * B;
          float* nNl = reinterpret_cast<float*>(nK + 3 * B);
          int* lvis = reinterpret_cast<int*>(lb + L.l_keys);
          const int TN = ls[LS_TN], N = ls[LS_N];
          const bool traced = ls[LS_TRACED] != 0;
          for (int r = ttid; r < nwin; r += TT) {
            const int wb = wins[r], c = wins[B + r];
            const float S = reinterpret_cast<const float*>(wins)[2 * B + r];
            const int Kb = mK[wb];
            const bool isnew = (c == Kb);
            if (isnew && Kb >= Kcap) {
              ls[LS_ERR] = 1;  // more clusters than the device tables hold
            } else {
              const TabEntry old = isnew ? TabEntry{kInitSlot, 0, 0, 0} : tab[(size_t)wb * Kcap + c];
              const bool moved = isnew || (c != mLast[wb]);
              const int lc = wcol[r];
              TabEntry nen;
              nen.slot = lcolnew[lc];
              nen.blocks = old.blocks + (moved ? 1 : 0);  // uisrnn.py:431-432; a new cluster starts at 1 (:76)
              nen.visits = old.visits + 1;
              nen.pad = 0;
              ntab[(size_t)r * Kcap + c] = nen;
              nK[r] = Kb + (isnew ? 1 : 0);
              atomicMax((int*)&misc[MI_MAXK], Kb + (isnew ? 1 : 0));
              nLast[r] = c;
              nTot[r] = mTot[wb] + (moved ? 1 : 0);
              nNl[r] = S;
              if (lcolsrc[lc] == old.slot) lvis[lc] = old.visits;  // same slot => same visit count
            }
            if (t >= TN - N) bp_cta[((size_t)g * p.maxN + (t - (TN - N))) * B + r] = ((unsigned)wb << 16) | (unsigned)c;
            if (traced) {
              const long long rows = ((long long)ls[LS_DBGROWS_HI] << 32) | (unsigned)ls[LS_DBGROWS_LO];
              if (p.dbg_win && rows + r < p.trace_capacity) {
                p.dbg_win[(rows + r) * 2 + 0] = wb;
                p.dbg_win[(rows + r) * 2 + 1] = c;
                p.dbg_score[rows + r] = S;
              }
              if (r == 0 && p.dbg_off) p.dbg_off[t + 1] = rows + nwin;
            }
          }
        }
      }
    }
    named_bar_sync(1, NT);  // every lane's M, winners and tables are published

    int nact = 0, Mtot = 0, colbase = 0;  // colbase: first CTA column of this thread's lane
    for (int g = 0; g < G; ++g) {
      nact += LSp(g)[LS_ACTIVE];
      if (g == team_of()) colbase = Mtot;
      Mtot += LSp(g)[LS_M];
    }
    if (nact == 0) break;
    // column list: lane-local -> CTA-wide, each team its own lane's columns
    if (team_of() < G) {
      const int g = team_of(), TT = (NW / G) * 32, ttid = tid - g * TT;
      volatile int* ls = LSp(g);
      const int M = ls[LS_M];
      const long long row = (((long long)ls[LS_ROW0_HI] << 32) | (unsigned)ls[LS_ROW0_LO]) + (ls[LS_T] % ls[LS_N]);
      const int* lcolsrc = reinterpret_cast<const int*>(lane_base(g) + L.l_lcol);
      const int* lvis = reinterpret_cast<const int*>(lane_base(g) + L.l_keys);
      for (int lc = ttid; lc < M; lc += TT) {
        const int f = colbase + lc;
        collane[f] = g;
        colsrc[f] = lcolsrc[lc];
        colnew[f] = lcolsrc[B + lc];
        colvis[f] = lvis[lc];
        colrow[f] = row;
      }
    }
    constexpr int kColsPerPass = TC ? TCN : C::CP;
    const int npass = TC ? (Mtot + kColsPerPass - 1) / kColsPerPass : max(1, (Mtot + C::CP - 1) / C::CP);
    if (tid == 0) {
      for (int g = 0; g < G; ++g) {
        volatile int* ls = LSp(g);
        if (ls[LS_ACTIVE]) { st_cand += ls[LS_NE]; st_steps += 1; }
      }
      st_cols += Mtot;
      st_pass += npass;
      if (!TC) { __threadfence_block(); misc[MI_PUBLISHED] = misc[MI_PUBLISHED] + npass; }  // the producer streams
    }
    named_bar_sync(1, NT);

    UIS_PHASE(0);
    // ---- P5: GRU + MLP for the Mtot distinct source states, C::CP columns per weight pass
    if constexpr (TC) {
      // Gaussian terms of the NEXT step, computed by every team for its lane while the tensor pipe works on the first
      // tiles of this pass: every slot of the next generation's tables except the ones this pass is about to write,
      // against x_{t+1} (uisrnn.py:411-414 reads the pre-update mean; slots are immutable once written).
      auto prescore = [&]() {
        if (team_of() < G) {
          const int g = team_of(), TW = NW / G, TT = TW * 32, ttid = tid - g * TT, twarp = warp - g * TW;
          volatile int* ls = LSp(g);
          unsigned* used = reinterpret_cast<unsigned*>(lane_base(g) + L.l_used);
          unsigned* scored = reinterpret_cast<unsigned*>(lane_base(g) + L.l_scored);
          cp_async_wait_all();  // x_{t+1} was requested in P0 by this team
          for (unsigned w = ttid; w < PW; w += TT) { used[w] = 0; scored[w] = 0; }  // (used: list marker)
          team_sync();
          const int nwin = ls[LS_NWIN];
          if (ls[LS_ACTIVE] && !ls[LS_ERR] && nwin > 0 && ls[LS_T] + 1 < ls[LS_TN]) {
            const int ngen = ls[LS_GEN] ^ 1;
            const int* nK = reinterpret_cast<const int*>(lane_base(g) + L.l_meta) + ngen * 4 * B;
            const TabEntry* ntab = reinterpret_cast<const TabEntry*>(lane_base(g) + L.l_tabs) + (size_t)ngen * B * Kcap;
            if (ttid == 0) atomicOr(scored, 1u);  // slot 0 = INIT (the new-cluster candidate)
            for (int f = ttid; f < nwin * Kcap; f += TT) {
              const int r = f / Kcap, c = f % Kcap;
              if (c < nK[r]) {
                const int slot = ntab[(size_t)r * Kcap + c].slot;
                atomicOr(scored + (slot >> 5), 1u << (slot & 31));
              }
            }
            team_sync();
            const int M = ls[LS_M];
            const int* lcolnew = reinterpret_cast<const int*>(lane_base(g) + L.l_lcol) + B;
            for (int lc = ttid; lc < M; lc += TT)  // the slots this step's passes write: scored in P1 of the next step
              atomicAnd(scored + (lcolnew[lc] >> 5), ~(1u << (lcolnew[lc] & 31)));
            team_sync();
            score_lane_slots(g, /*against the next frame=*/true, ttid, twarp, TW);
          }
        }
        named_bar_sync(1, NT);  // the warpgroups enter the pass's tiles together
      };
      auto nothing = []() {};
      if (Mtot == 0 && team_of() < G) {  // no pass, no pre-scoring: every team clears its own lane's marks
        const int g = team_of(), TT = (NW / G) * 32;
        for (unsigned w = tid - g * TT; w < PW; w += TT) reinterpret_cast<unsigned*>(lane_base(g) + L.l_scored)[w] = 0;
      }
      for (int m0 = 0; m0 < Mtot; m0 += TCN) {
        if (m0 == 0)
          tc_run_pass<H, D, TC ? TCN : 16>(p, reinterpret_cast<const unsigned char*>(ring), reinterpret_cast<unsigned char*>(XA),
                                           tb, tc_boxes, cc, m0, min(TCN, Mtot - m0), pool_mean_cta, pool_hidden_cta,
                                           tc_scratch_cta, tid, lane, warp, ph, tmark, ph + 16, prescore);
        else
          tc_run_pass<H, D, TC ? TCN : 16>(p, reinterpret_cast<const unsigned char*>(ring), reinterpret_cast<unsigned char*>(XA),
                                           tb, tc_boxes, cc, m0, min(TCN, Mtot - m0), pool_mean_cta, pool_hidden_cta,
                                           tc_scratch_cta, tid, lane, warp, ph, tmark, ph + 16, nothing);
        named_bar_sync(1, NT);
        UIS_PHASE(4);
      }
    } else {
    if (Mtot == 0 && !STAT) drain_pass<C>(full, empty, it, lane, p.depth, xsize);
    for (int m0 = 0; m0 < Mtot; m0 += C::CP) {
      const int Mp = min(C::CP, Mtot - m0);
      // gather the source hidden states, transposed: XA[k][m]
#pragma unroll
      for (int u = 0; u < UPT; ++u) {
        const int j = tid + NT * u;
#pragma unroll
        for (int c = 0; c < C::CP / 4; ++c) {
          float hv[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const int m = 4 * c + q;
            const float* hp = pool_hidden_cta + (size_t)collane[m0 + m] * pool_h_stride + (size_t)colsrc[m0 + m] * DH + j;
            hv[q] = (m < Mp) ? (STAT ? __ldcg(hp) : *hp) : 0.f;
          }
          reinterpret_cast<float4*>(XA + (size_t)j * C::CP)[c] = make_float4(hv[0], hv[1], hv[2], hv[3]);
        }
      }
      named_bar_sync(1, NT);
      UIS_PHASE(1);
      if constexpr (STAT)
        stat_pass<H, D, C::CP, NT>(p, ring, XA, XB, cc, m0, Mp, pool_mean_cta, pool_hidden_cta,
                                   p.stat_scratch + (size_t)sgroup * C::CP * H, p.stat_bar + (size_t)sgroup * kStatGroup, stat_epoch, sq, tid, ph, tmark);
      else run_pass_any<C, DEEP, XCL>(p, ring, full, empty, it, XA, XB, cc, m0, Mp, pool_mean_cta, pool_hidden_cta, bh, b1r, b2r, tid, lane, ph, tmark, &xc);
      named_bar_sync(1, NT);
      UIS_PHASE(4);
    }
    }  // !TC

    // ---- P6: every team advances its lane; a finished utterance is back-tracked and replaced
    if (team_of() < G) {
      const int g = team_of(), TT = (NW / G) * 32, ttid = tid - g * TT;
      volatile int* ls = LSp(g);
      const bool act = ls[LS_ACTIVE] != 0;
      const bool fin = act && (ls[LS_ERR] != 0 || ls[LS_NWIN] == 0 || ls[LS_T] + 1 >= ls[LS_TN]);
      if (fin) {  // debug taps and outputs of the finishing utterance (the team)
        const int u = ls[LS_U], nwin = ls[LS_NWIN], ngen = ls[LS_GEN] ^ 1;
        const bool ok = !ls[LS_ERR] && nwin > 0;
        const int* fK = reinterpret_cast<const int*>(lane_base(g) + L.l_meta) + ngen * 4 * B;
        const float* fNl = reinterpret_cast<const float*>(fK + 3 * B);
        // utterance epilogue: back-track the returned hypotheses (uisrnn.py:561), one per thread.  Hypothesis j is the
        // j-th final rank with min_speakers clusters (rank 0 when none has them, j = 0); it walks its own column chain
        // into label plane j.  (Stationary-weights mode: the replicas of a group decode the same utterance, and CTA 0
        // of the group reports it.)
        for (int j = ttid; j < p.n_best && !(STAT && sq != 0); j += TT) {
          const int r0 = ok ? nbest_rank(fK, nwin, ls[LS_KLO], j) : -1;
          const int N = ls[LS_N];
          int* lab = p.labels + ((size_t)(u / p.n_utt) * p.n_best + j) * p.label_plane +
                     (((long long)ls[LS_ROW0_HI] << 32) | (unsigned)ls[LS_ROW0_LO]);
          if (r0 < 0) {
            for (int i = 0; i < N; ++i) lab[i] = -1;
          } else {
            const unsigned* bp = bp_cta + (size_t)g * p.maxN * B;
            int r = r0;
            for (int i = N - 1; i >= 0; --i) {
              const unsigned e = bp[(size_t)i * B + r];
              lab[i] = (int)(e & 0xffffu);
              r = (int)(e >> 16);
            }
          }
          if (j == 0) {
            if (p.spk_out) p.spk_out[u] = ok ? fK[r0] : 0;
            if (p.nbest_count) p.nbest_count[u] = ok ? nbest_n(fK, nwin, ls[LS_KLO], p.n_best) : 0;
          }
          nbest_store(p, u, j, r0, fK, fNl);
        }
        if (p.dbg_final_scores && tap_leader) {
          for (int b = ttid; b < B; b += TT) p.dbg_final_scores[(size_t)u * B + b] = (ok && b < nwin) ? fNl[b] : INF;
          if (ttid == 0 && p.dbg_final_k) p.dbg_final_k[u] = ok ? fK[0] : 0;
        }
        if (ls[LS_TRACED] && ok && p.dbg_best_mean) {
          // (stationary-weights mode: the slots are in the group's pool, published by the group barrier that ended the
          //  last weight pass; other CTAs wrote most of them, so the reads bypass L1)
          const TabEntry* ftab = reinterpret_cast<const TabEntry*>(lane_base(g) + L.l_tabs) + (size_t)ngen * B * Kcap;
          for (int c = 0; c < fK[0]; ++c) {  // best hypothesis = rank 0
            const TabEntry en = ftab[c];
            const float* mp = pool_mean_cta + g * pool_m_stride + (size_t)en.slot * D;
            const float* hp = pool_hidden_cta + g * pool_h_stride + (size_t)en.slot * DH;
            for (int d = ttid; d < D; d += TT) p.dbg_best_mean[(size_t)c * D + d] = STAT ? __ldcg(mp + d) : mp[d];
            for (int q = ttid; q < DH; q += TT) p.dbg_best_hidden[(size_t)c * DH + q] = STAT ? __ldcg(hp + q) : hp[q];
            if (ttid == 0) p.dbg_best_blocks[c] = en.blocks;
          }
        }
        if constexpr (STAT) {
          // The traced utterance's state is read from the group's pool above; the other CTAs may only write the slots
          // of their next utterance (its first weight pass, before any group barrier) once the leader has read it.
          // (One lane per CTA in this mode: the team is every consumer thread.)
          if (u == p.trace_utt && p.dbg_best_mean)
            stat_group_sync<NT>(p.stat_bar + (size_t)sgroup * kStatGroup, stat_epoch, tid);
        }
      }
      team_sync();  // the finished lane's tables are read before lane_fetch reuses them
      if (ttid == 0 && act) {
        if (fin) {
          if (!(STAT && sq != 0)) p.status[ls[LS_U]] = ls[LS_ERR] ? -4 : ls[LS_NWIN] == 0 ? -1 : 0;
          lane_fetch(g);
        } else {
          const long long rows = (((long long)ls[LS_DBGROWS_HI] << 32) | (unsigned)ls[LS_DBGROWS_LO]) + ls[LS_NWIN];
          ls[LS_DBGROWS_LO] = (int)(rows & 0xffffffffll); ls[LS_DBGROWS_HI] = (int)(rows >> 32);
          ls[LS_T] = ls[LS_T] + 1; ls[LS_NB] = ls[LS_NWIN]; ls[LS_GEN] = ls[LS_GEN] ^ 1; ls[LS_FRESH] = 0;
        }
      }
      team_sync();
      if (fin && ls[LS_ACTIVE] && ls[LS_FRESH]) {
        lane_prefetch(g, 0, ttid, TT);
        cp_async_commit();
      }
    }
    UIS_PHASE(5);
  }  // CTA steps

  cp_async_wait_all();
  if constexpr (XCL) xch_barrier<NT>(xc, tid);  // peers may still be reading this CTA's exchange buffer
  if (tid == 0) {
    __threadfence_block();
    misc[MI_DONE] = 1;
    if (XCL && xc.rank != 0) return;  // the replicas of a cluster count once
    if (STAT && sq != 0) return;
    atomicAdd(&p.stats[0], (unsigned long long)st_cols);
    atomicAdd(&p.stats[1], (unsigned long long)st_pass);
    atomicAdd(&p.stats[2], (unsigned long long)st_cand);
    atomicAdd(&p.stats[3], (unsigned long long)st_steps);
    atomicMax(&p.stats[4], (unsigned long long)max(st_maxk, (long long)misc[MI_MAXK]));
    for (int i = 0; i < 10; ++i) atomicAdd(&p.stats[8 + i], (unsigned long long)ph[i]);
    if constexpr (TC)
      for (int i = 0; i < 4; ++i) atomicAdd(&p.stats[18 + i], (unsigned long long)ph[16 + i]);
  }
}

}  // namespace uis
