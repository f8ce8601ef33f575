// Beam search with look_ahead >= 2 (one utterance per CTA), sm_90a.
//
// Reference semantics: uisrnn/uisrnn.py:455-477 (_calculate_score enumerates every index tuple
// (c_1..c_L), c_i <= K + #clusters opened earlier in the tuple), :388-453 (each sub-step is scored
// on the state left by the previous sub-steps), :529-561 (rank all tuples of all hypotheses,
// rebuild the best beam_size).  Work is organised as a prefix tree per beam step:
//   level i node  = a valid prefix (c_1..c_i) of one hypothesis; it stores only what differs from
//                   its parent: the (slot, blocks, visits) of cluster c_i, K, total blocks, score;
//   levels < L'   : every node is evaluated (GRU + MLP on frame i) because deeper scores need its
//                   updated mean / hidden state; nodes sharing a source slot share the evaluation;
//   level L'      : leaves are only scored (the last sub-step's GRU never enters a score),
//                   ranked with the reference's flat-index tie-break, and the best beam_size are
//                   evaluated and materialised as the next generation of hypothesis tables.
// The weight streaming / register-tiled FFMA passes are the ones of uis_beam.cuh (run_pass).
#pragma once
#include "uis_beam.cuh"

namespace uis {

struct TreeLayout {
  unsigned ring, xa, xb, wv, xt, tabs, meta, n_parent, n_c, n_nl, n_k, n_tot, n_ov, lvl, l_pc, l_key, colsrc, colnew, colvis, colrow, collane, colmap, used, wins, bars, misc, total;
};

template <int H, int D>
__host__ __device__ inline TreeLayout make_tree_layout(int B, int Kcap, int L, int NI, int NLF, int P) {
  constexpr int kCP = tree_cp<H>();
  TreeLayout T;
  unsigned o = 0;
  T.ring = o;     o += kStages * kStageBytes;
  T.xa = o;       o += H * kCP * 4;
  T.xb = o;       o += H * kCP * 4;
  T.wv = o;       o += D * 4;
  T.xt = o;       o += (unsigned)L * D * 4;
  T.tabs = o;     o += 2u * B * Kcap * 16;
  T.meta = o;     o += 2u * 4 * B * 4;
  T.n_parent = o; o += align_up((unsigned)NI * 4, 16);
  T.n_c = o;      o += align_up((unsigned)NI * 4, 16);
  T.n_nl = o;     o += align_up((unsigned)NI * 4, 16);
  T.n_k = o;      o += align_up((unsigned)NI * 4, 16);
  T.n_tot = o;    o += align_up((unsigned)NI * 4, 16);
  T.n_ov = o;     o += (unsigned)NI * 16;
  T.lvl = o;      o += 64;
  T.l_pc = o;     o += align_up((unsigned)NLF * 4, 16);   // (parent << 8) | cluster
  T.l_key = o;    o += align_up((unsigned)NLF * 8, 16);   // score (ordered bits) << 32 | flat index
  T.colsrc = o;   o += align_up((unsigned)NI * 4, 16);
  T.colnew = o;   o += align_up((unsigned)NI * 4, 16);
  T.colvis = o;   o += align_up((unsigned)NI * 4, 16);
  T.colrow = o;   o += align_up((unsigned)NI * 8, 16);
  T.collane = o;  o += align_up((unsigned)NI * 4, 16);
  T.colmap = o;   o += align_up((unsigned)P * 4, 16);
  T.used = o;     o += align_up(((unsigned)P + 31) / 32 * 4, 16);
  T.wins = o;     o += align_up((unsigned)B * 4, 16);
  T.bars = o;     o += 2 * kStages * 8;
  T.misc = o;     o += 64;
  T.total = o;
  return T;
}

// Spill policy: the arrays whose size follows the tree (nodes, leaves, columns, slot map and free bitmap) live in a
// per-CTA arena in device memory; everything else keeps its shared-memory place (make_tree_layout with no nodes).
struct TreeArena {
  size_t n_parent, n_c, n_nl, n_k, n_tot, n_ov, l_pc, l_key, colsrc, colnew, colvis, colrow, collane, colmap, used, total;
};

__host__ __device__ inline TreeArena make_tree_arena(int NI, int NLF, int P) {
  TreeArena A;
  size_t o = 0;
  const size_t ni = (size_t)NI, nl = (size_t)NLF, np = (size_t)P;
  auto take = [&](size_t bytes) { const size_t at = o; o += (bytes + 127) / 128 * 128; return at; };
  A.n_parent = take(ni * 4); A.n_c = take(ni * 4); A.n_nl = take(ni * 4); A.n_k = take(ni * 4); A.n_tot = take(ni * 4);
  A.n_ov = take(ni * 16);
  A.l_pc = take(nl * 4); A.l_key = take(nl * 8);
  A.colsrc = take(ni * 4); A.colnew = take(ni * 4); A.colvis = take(ni * 4); A.colrow = take(ni * 8); A.collane = take(ni * 4);
  A.colmap = take(np * 4); A.used = take((np + 31) / 32 * 4);
  A.total = o;
  return A;
}

// Shared scratch of the spill kernel, after make_tree_layout(..).total: the survivors of the leaf selection
// (<= 32 keys), the 256-bucket radix histogram, the warp totals of the block scan and 4 broadcast words.
constexpr unsigned kTreeSpillScratch = 32 * 8 + 256 * 4 + 36 * 4 + 4 * 4;

// Exclusive prefix sum of v over the NT consumer threads; *total = the sum of all.  sc: >= 33 ints of shared memory.
template <int NT>
__device__ __forceinline__ int block_excl_scan(int v, int* sc, int* total, int lane, int warp) {
  int incl = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
  if (lane == 31) sc[warp] = incl;
  named_bar_sync(1, NT);
  if (warp == 0) {
    const int w = (lane < NT / 32) ? sc[lane] : 0;
    int wi = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, wi, o); if (lane >= o) wi += t; }
    sc[lane] = wi - w;
    if (lane == 31) sc[32] = wi;
  }
  named_bar_sync(1, NT);
  const int r = sc[warp] + incl - v;
  *total = sc[32];
  named_bar_sync(1, NT);
  return r;
}

// Leaf positions of the nwin (1..32) smallest of the n unique keys, in ascending key order, into wins[0..nwin).
// MSD radix select over 8-bit digits finds the nwin-th smallest key; the nwin keys at or below it are then ranked.
// Any exact selection of unique keys gives what the on-chip counting rank gives.
template <int NT>
__device__ void tree_select_smallest(const unsigned long long* key, int n, int nwin, int* wins, unsigned char* scratch,
                                     int tid, int lane, int warp) {
  unsigned long long* surv = reinterpret_cast<unsigned long long*>(scratch);
  unsigned* hist = reinterpret_cast<unsigned*>(scratch + 32 * 8);
  volatile int* sel = reinterpret_cast<volatile int*>(scratch + 32 * 8 + 256 * 4 + 36 * 4);
  unsigned long long prefix = 0, mask = 0;
  int k = nwin;  // rank of the nwin-th smallest key among the keys that equal `prefix` under `mask`
  for (int shift = 56; shift >= 0; shift -= 8) {
    for (int i = tid; i < 256; i += NT) hist[i] = 0;
    named_bar_sync(1, NT);
    for (int f0 = warp * 32; f0 < n; f0 += NT) {
      const int f = f0 + lane;
      unsigned d = 256;
      if (f < n) { const unsigned long long x = key[f]; if ((x & mask) == prefix) d = (unsigned)(x >> shift) & 255u; }
      const unsigned peers = __match_any_sync(0xffffffffu, d);
      if (d < 256 && lane == __ffs(peers) - 1) atomicAdd(&hist[d], (unsigned)__popc(peers));
    }
    named_bar_sync(1, NT);
    if (warp == 0) {  // the bucket that holds the k-th key: lane l owns buckets 8l .. 8l+7
      unsigned c[8];
      int s = 0;
#pragma unroll
      for (int i = 0; i < 8; ++i) { c[i] = hist[8 * lane + i]; s += (int)c[i]; }
      int incl = s;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
      const int excl = incl - s;
      if (excl < k && k <= incl) {
        int cum = excl;
        for (int i = 0; i < 8; ++i) {
          if (cum + (int)c[i] >= k) { sel[0] = 8 * lane + i; sel[1] = k - cum; sel[2] = (int)c[i]; break; }
          cum += (int)c[i];
        }
      }
    }
    named_bar_sync(1, NT);
    prefix |= (unsigned long long)sel[0] << shift;
    mask |= 255ull << shift;
    k = sel[1];
    if (sel[2] == 1) break;  // the nwin-th smallest key is the only one with this prefix
  }
  // the keys below `prefix` under `mask` plus the one equal to it: exactly the nwin smallest
  if (tid == 0) sel[3] = 0;
  named_bar_sync(1, NT);
  for (int f = tid; f < n; f += NT) {
    const unsigned long long x = key[f];
    if ((x & mask) <= prefix) {
      const int s = atomicAdd((int*)&sel[3], 1);
      if (s < nwin) surv[s] = x;
    }
  }
  named_bar_sync(1, NT);
  if (tid < nwin) {
    const unsigned long long x = surv[tid];
    int rank = 0;
    for (int q = 0; q < nwin; ++q) rank += (surv[q] < x) ? 1 : 0;
    wins[rank] = (int)(unsigned)x;  // low 32 bits: the leaf position
  }
}

enum { TM_PUBLISHED = 0, TM_DONE, TM_UIDX, TM_ERR, TM_NFINITE, TM_M, TM_COUNT, TM_NWIN };

// SPILL = false: the whole tree of a beam step lives in shared memory (node_cap / leaf_cap sized by the host to what
// fits), and an utterance whose tree outgrows it ends with status -5.  SPILL = true: the tree-sized arrays live in a
// device-memory arena of node_cap / leaf_cap entries per CTA (p.tree_arena), and the kernel decodes only the
// utterances left at status -5 by the shared-memory kernel (all of them with p.tree_spill_all).
template <int H, int D, bool DEEP, bool SPILL = false>
__global__ void __launch_bounds__(Cfg<H, D, tree_cp<H>()>::BLOCK, 1) uis_beam_tree_kernel(const BeamParams p) {
  using C = Cfg<H, D, tree_cp<H>()>;
  constexpr int NT = C::NT, NW = C::NW, UPT = C::UPT;
  extern __shared__ __align__(128) unsigned char smem[];
  const int B = p.B, Kcap = p.Kcap, L = p.L, NI = p.node_cap, NLF = p.leaf_cap;
  const TreeLayout T = make_tree_layout<H, D>(B, Kcap, L, SPILL ? 0 : NI, SPILL ? 0 : NLF, SPILL ? 0 : p.P);
  float* ring = reinterpret_cast<float*>(smem + T.ring);
  float* XA = reinterpret_cast<float*>(smem + T.xa);
  float* XB = reinterpret_cast<float*>(smem + T.xb);
  float* wv = reinterpret_cast<float*>(smem + T.wv);
  float* xt = reinterpret_cast<float*>(smem + T.xt);
  TabEntry* tabs = reinterpret_cast<TabEntry*>(smem + T.tabs);
  int* meta = reinterpret_cast<int*>(smem + T.meta);
  int* n_parent = reinterpret_cast<int*>(smem + T.n_parent);
  int* n_c = reinterpret_cast<int*>(smem + T.n_c);
  float* n_nl = reinterpret_cast<float*>(smem + T.n_nl);
  int* n_k = reinterpret_cast<int*>(smem + T.n_k);
  int* n_tot = reinterpret_cast<int*>(smem + T.n_tot);
  TabEntry* n_ov = reinterpret_cast<TabEntry*>(smem + T.n_ov);
  int* lvl = reinterpret_cast<int*>(smem + T.lvl);  // lvl[i] = first node of level i (1-based), lvl[i+1] = end
  unsigned* l_pc = reinterpret_cast<unsigned*>(smem + T.l_pc);
  unsigned long long* l_key = reinterpret_cast<unsigned long long*>(smem + T.l_key);
  int* colsrc = reinterpret_cast<int*>(smem + T.colsrc);
  int* colnew = reinterpret_cast<int*>(smem + T.colnew);
  int* colvis = reinterpret_cast<int*>(smem + T.colvis);
  long long* colrow = reinterpret_cast<long long*>(smem + T.colrow);
  int* collane = reinterpret_cast<int*>(smem + T.collane);
  int* colmap = reinterpret_cast<int*>(smem + T.colmap);
  unsigned* used = reinterpret_cast<unsigned*>(smem + T.used);
  int* wins = reinterpret_cast<int*>(smem + T.wins);
  if constexpr (SPILL) {  // the tree-sized arrays move to this CTA's arena
    const TreeArena A = make_tree_arena(NI, NLF, p.P);
    unsigned char* const ar = p.tree_arena + (size_t)blockIdx.x * A.total;
    n_parent = reinterpret_cast<int*>(ar + A.n_parent);
    n_c = reinterpret_cast<int*>(ar + A.n_c);
    n_nl = reinterpret_cast<float*>(ar + A.n_nl);
    n_k = reinterpret_cast<int*>(ar + A.n_k);
    n_tot = reinterpret_cast<int*>(ar + A.n_tot);
    n_ov = reinterpret_cast<TabEntry*>(ar + A.n_ov);
    l_pc = reinterpret_cast<unsigned*>(ar + A.l_pc);
    l_key = reinterpret_cast<unsigned long long*>(ar + A.l_key);
    colsrc = reinterpret_cast<int*>(ar + A.colsrc);
    colnew = reinterpret_cast<int*>(ar + A.colnew);
    colvis = reinterpret_cast<int*>(ar + A.colvis);
    colrow = reinterpret_cast<long long*>(ar + A.colrow);
    collane = reinterpret_cast<int*>(ar + A.collane);
    colmap = reinterpret_cast<int*>(ar + A.colmap);
    used = reinterpret_cast<unsigned*>(ar + A.used);
  }
  unsigned char* const spill_scratch = smem + T.total;  // kTreeSpillScratch bytes, SPILL only
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + T.bars);
  uint64_t* empty = full + kStages;
  volatile int* misc = reinterpret_cast<volatile int*>(smem + T.misc);

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) {
    for (int s = 0; s < kStages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], NW); }
    for (int i = 0; i < 16; ++i) misc[i] = 0;
    fence_mbar_init();
  }
  __syncthreads();
  if (warp >= NW) {
    if constexpr (C::REBALANCE) asm volatile("setmaxnreg.dec.sync.aligned.u32 24;");
    if (warp == NW && lane == 0) producer_loop<C>(p, ring, full, empty, misc);
    return;
  }
  if constexpr (C::REBALANCE) asm volatile("setmaxnreg.inc.sync.aligned.u32 240;");

  const int DH = p.depth * H;
  const size_t pool_m_stride = (size_t)p.P * D, pool_h_stride = (size_t)p.P * DH;
  float* pool_mean = p.pool_mean + (size_t)blockIdx.x * pool_m_stride;
  float* pool_hidden = p.pool_hidden + (size_t)blockIdx.x * pool_h_stride;
  unsigned* bp_lab = p.bp + (size_t)blockIdx.x * ((size_t)p.maxTN + p.maxSteps) * B;  // [frame][r] cluster
  unsigned* bp_par = bp_lab + (size_t)p.maxTN * B;                                      // [step][r] parent rank
  const unsigned PW = (unsigned)(p.P + 31) / 32;
  const float INF = __int_as_float(0x7f800000);

  float bh[C::RG], b1r[UPT];
#pragma unroll
  for (int i = 0; i < C::RG; ++i) bh[i] = p.bhh[(i / UPT) * H + tid + NT * (i % UPT)];
#pragma unroll
  for (int u = 0; u < UPT; ++u) b1r[u] = p.b1[tid + NT * u];
  const float b2r = (tid < D) ? p.b2[tid] : 0.f;
  if (tid < D) { wv[tid] = p.wvec[tid]; pool_mean[(size_t)kInitSlot * D + tid] = p.mean0[tid]; }
  for (int q = tid; q < DH; q += NT) pool_hidden[(size_t)kInitSlot * DH + q] = p.hidden0[q];
  for (int i = tid; i < NI; i += NT) collane[i] = 0;
  const ColCtx cc{collane, colsrc, colnew, colvis, colrow};

  unsigned it = 0;
  unsigned long long st_cols = 0, st_pass = 0, st_cand = 0, st_steps = 0;
  int st_maxk = 0;
  long long ph_dummy[10];
  long long tmark_dummy = 0;

  // (slot, blocks, visits) of cluster c in the state reached by node `n` of level `level`
  // (level 0: n is a hypothesis index of the current generation).
  auto lookup = [&](int level, int n, int c, const TabEntry* tab, const int* mK) -> TabEntry {
    while (level >= 1) {
      if (n_c[n] == c) return n_ov[n];
      n = n_parent[n];
      --level;
    }
    return (c < mK[n]) ? tab[(size_t)n * Kcap + c] : TabEntry{kInitSlot, 0, 0, 0};
  };

  // GRU + MLP evaluation of nodes [a, b) (frame index fi of the chunk): columns are the distinct
  // source slots; on return n_ov[node] is the post-update entry.
  auto evaluate = [&](int a, int b, long long girow) {
    for (int s = tid; s < p.P; s += NT) colmap[s] = 0;
    named_bar_sync(1, NT);
    for (int n = a + tid; n < b; n += NT) colmap[n_ov[n].slot] = 1;
    named_bar_sync(1, NT);
    if (warp == 0) {
      // column ids for flagged slots (ascending slot order) and new slots from the free bitmap
      int cnt = 0;
      for (int s = lane; s < p.P; s += 32) cnt += colmap[s] ? 1 : 0;
      int incl = cnt;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
      const int M = __shfl_sync(0xffffffffu, incl, 31);
      int idx = incl - cnt;
      // interleaved ownership (s = lane + 32k) => ids are unique but not slot-ordered; any bijection will do
      for (int s = lane; s < p.P; s += 32)
        if (colmap[s]) { colsrc[idx] = s; colmap[s] = idx + 1; ++idx; }
      int fcnt = 0;
      for (unsigned w = lane; w < PW; w += 32) {
        unsigned fr = ~used[w];
        if (w == PW - 1 && (p.P & 31)) fr &= (1u << (p.P & 31)) - 1;
        fcnt += __popc(fr);
      }
      int fincl = fcnt;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, fincl, o); if (lane >= o) fincl += v; }
      const int nfree = __shfl_sync(0xffffffffu, fincl, 31);
      int fidx = fincl - fcnt;
      for (unsigned w = lane; w < PW && fidx < M; w += 32) {
        unsigned fr = ~used[w];
        if (w == PW - 1 && (p.P & 31)) fr &= (1u << (p.P & 31)) - 1;
        unsigned taken = 0;
        while (fr && fidx < M) {
          const int bit = __ffs(fr) - 1;
          fr &= fr - 1;
          taken |= 1u << bit;
          colnew[fidx++] = (int)(w * 32 + bit);
        }
        used[w] |= taken;  // temporaries stay reserved until the end of the beam step
      }
      if (lane == 0) { misc[TM_M] = M; if (nfree < M || M > NI) misc[TM_ERR] = 2; }
    }
    named_bar_sync(1, NT);
    const int M = misc[TM_M];
    for (int n = a + tid; n < b; n += NT) {
      const int col = colmap[n_ov[n].slot] - 1;
      colvis[col] = n_ov[n].visits;  // same source slot => same visit count
    }
    for (int m = tid; m < M; m += NT) colrow[m] = girow;
    const int npass = (M + C::CP - 1) / C::CP;
    if (tid == 0 && npass > 0) {
      st_cols += M; st_pass += npass;
      __threadfence_block();
      misc[TM_PUBLISHED] = misc[TM_PUBLISHED] + npass;
    }
    named_bar_sync(1, NT);
    if (misc[TM_ERR]) {  // keep the producer protocol consistent, skip the math
      for (int q = 0; q < npass; ++q) drain_pass<C>(full, empty, it, lane, p.depth);
      return;
    }
    for (int m0 = 0; m0 < M; m0 += C::CP) {
      const int Mp = min(C::CP, M - m0);
#pragma unroll
      for (int u = 0; u < UPT; ++u) {
        const int j = tid + NT * u;
#pragma unroll
        for (int c4 = 0; c4 < C::CP / 4; ++c4) {
          float hv[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const int m = 4 * c4 + q;
            hv[q] = (m < Mp) ? pool_hidden[(size_t)colsrc[m0 + m] * DH + j] : 0.f;
          }
          reinterpret_cast<float4*>(XA + (size_t)j * C::CP)[c4] = make_float4(hv[0], hv[1], hv[2], hv[3]);
        }
      }
      named_bar_sync(1, NT);
      run_pass_any<C, DEEP>(p, ring, full, empty, it, XA, XB, cc, m0, Mp, pool_mean, pool_hidden, bh, b1r, b2r, tid, lane, ph_dummy, tmark_dummy);
      named_bar_sync(1, NT);
    }
    for (int n = a + tid; n < b; n += NT) {
      TabEntry e = n_ov[n];
      e.slot = colnew[colmap[e.slot] - 1];
      e.visits += 1;
      n_ov[n] = e;
    }
    named_bar_sync(1, NT);
  };

  for (;;) {
    if (tid == 0) misc[TM_UIDX] = atomicAdd(p.queue, 1);
    named_bar_sync(1, NT);
    const int uidx = misc[TM_UIDX];
    if (uidx >= p.U) break;
    const int u = p.order[uidx], utt = u % p.n_utt;  // u: the job
    if constexpr (SPILL) {  // decoded by the shared-memory kernel (or failed there for another reason)
      if (!p.tree_spill_all && p.status[u] != -5) { named_bar_sync(1, NT); continue; }
    }
    const long long row0 = p.row_off[utt];
    const int N = (int)(p.row_off[utt + 1] - row0);
    const int TN = p.T * N;
    const bool traced = (u == p.trace_utt);
    long long dbg_rows = 0;
    int gen = 0, nb = 1;
    if (tid == 0) {
      meta[0] = 0; meta[B] = -1; meta[2 * B] = 0; reinterpret_cast<float*>(meta)[3 * B] = 0.f;
      misc[TM_ERR] = 0;
      if (traced && p.dbg_off) p.dbg_off[0] = 0;
    }
    named_bar_sync(1, NT);
    bool failed = false;
    int step = 0;

    for (int t0 = 0; t0 < TN; t0 += L, ++step) {
      const int Lc = min(L, TN - t0);
      int* mK = meta + gen * 4 * B; int* mLast = mK + B; int* mTot = mK + 2 * B;
      float* mNl = reinterpret_cast<float*>(mK + 3 * B);
      int* nK = meta + (gen ^ 1) * 4 * B; int* nLast = nK + B; int* nTot = nK + 2 * B;
      float* nNl = reinterpret_cast<float*>(nK + 3 * B);
      const TabEntry* tab = tabs + (size_t)gen * B * Kcap;
      TabEntry* ntab = tabs + (size_t)(gen ^ 1) * B * Kcap;

      // frames of this chunk; live-slot bitmap from the current generation
      for (int q = tid; q < Lc * (D / 4); q += NT) {
        const int i = q / (D / 4), d4 = q % (D / 4);
        reinterpret_cast<float4*>(xt + (size_t)i * D)[d4] =
            reinterpret_cast<const float4*>(p.x + (size_t)(row0 + (t0 + i) % N) * D)[d4];
      }
      for (unsigned w = tid; w < PW; w += NT) used[w] = (w == 0) ? 1u : 0u;
      named_bar_sync(1, NT);
      for (int q = tid; q < nb * Kcap; q += NT) {
        const int b = q / Kcap, c = q % Kcap;
        if (c < mK[b]) { const int s = tab[(size_t)b * Kcap + c].slot; atomicOr(&used[s >> 5], 1u << (s & 31)); }
      }
      int kmax = 0;
      for (int b = 0; b < nb; ++b) kmax = max(kmax, mK[b]);
      if (tid == 0) { lvl[0] = 0; lvl[1] = 0; }
      named_bar_sync(1, NT);

      int n_leaves = 0;
      for (int level = 1; level <= Lc; ++level) {
        const bool last = (level == Lc);
        const int pa = (level == 1) ? 0 : lvl[level - 1], pb = (level == 1) ? nb : lvl[level];
        if constexpr (SPILL) {
          // children offsets: block-wide prefix sum over the parents' K + 1 fan-outs, NT parents at a time
          const int base = lvl[level];
          const int cap = last ? NLF : NI - base;
          int* sc = reinterpret_cast<int*>(spill_scratch + 32 * 8 + 256 * 4);
          int tot = 0;
          for (int q0 = pa; q0 < pb; q0 += NT) {
            const int q = q0 + tid;
            const int Kp = (q < pb) ? ((level == 1) ? mK[q] : n_k[q]) : -1;
            const int fan = Kp + (Kp < spk_max(p, utt) ? 1 : 0);  // at max_speakers: no new-cluster child
            int chunk;
            const int o = tot + block_excl_scan<NT>(fan, sc, &chunk, lane, warp);
            if (chunk > cap - tot) { if (tid == 0) misc[TM_ERR] = 3; break; }
            for (int c = 0; c < fan; ++c) {
              if (last) l_pc[o + c] = ((unsigned)q << 8) | (unsigned)c;
              else { n_parent[base + o + c] = q; n_c[base + o + c] = c; }
            }
            tot += chunk;
          }
          if (tid == 0) {
            misc[TM_COUNT] = tot;
            if (!last) lvl[level + 1] = base + tot;
            st_cand += tot;
          }
        } else if (tid == 0) {  // children offsets (serial over parents; at most a few hundred)
          int tot = 0;
          const int base = lvl[level];
          for (int q = pa; q < pb; ++q) {
            const int Kp = (level == 1) ? mK[q] : n_k[q];
            const int fan = Kp + (Kp < spk_max(p, utt) ? 1 : 0);  // at max_speakers: no new-cluster child
            const int cap = last ? NLF : NI - base;
            if (tot + fan > cap) { misc[TM_ERR] = 3; break; }
            for (int c = 0; c < fan; ++c) {
              if (last) l_pc[tot + c] = ((unsigned)q << 8) | (unsigned)c;
              else { n_parent[base + tot + c] = q; n_c[base + tot + c] = c; }
            }
            tot += fan;
          }
          misc[TM_COUNT] = tot;
          if (!last) lvl[level + 1] = base + tot;
          st_cand += tot;
        }
        named_bar_sync(1, NT);
        if (misc[TM_ERR]) break;
        const int count = misc[TM_COUNT];
        const int base = lvl[level];
        const float* xs = xt + (size_t)(level - 1) * D;
        // score every child: one warp each (all lanes resolve the same indices)
        for (int f = warp; f < count; f += NW) {
          const int par = last ? (int)(l_pc[f] >> 8) : n_parent[base + f];
          const int c = last ? (int)(l_pc[f] & 255u) : n_c[base + f];
          int Kp, lastp, totp; float nlp;
          if (level == 1) { Kp = mK[par]; lastp = mLast[par]; totp = mTot[par]; nlp = mNl[par]; }
          else { Kp = n_k[par]; lastp = n_c[par]; totp = n_tot[par]; nlp = n_nl[par]; }
          const bool isnew = (c == Kp);
          const TabEntry en = isnew ? TabEntry{kInitSlot, 0, 0, 0} : lookup(level - 1, par, c, tab, mK);
          const float* mu = pool_mean + (size_t)en.slot * D;
          float4 m4[1][(D + 127) / 128];
#pragma unroll
          for (int i = 0; i < (D + 127) / 128; ++i)
            if (lane * 4 + i * 128 < D) m4[0][i] = *reinterpret_cast<const float4*>(mu + lane * 4 + i * 128);
          const bool live[1] = {true};
          const float acc = gauss_rows<D, 1>(m4, live, xs, wv, lane);
          if (lane == 0) {
            const JobLogs lg = job_logs(p, u / p.n_utt);
            double pen;
            if (!isnew) pen = (c == lastp) ? lg.log_1mp0 : (lg.log_p0 + __ldg(p.logn + en.blocks)) - __ldg(lg.logtot + totp);
            else pen = (lg.log_p0 + lg.log_alpha) - __ldg(lg.logtot + totp);
            const float loss = __double2float_rn((double)acc - pen);
            const float S = __fadd_rn(nlp, loss);  // per sub-step fp32 accumulation (uisrnn.py:452)
            if (last) {
              l_key[f] = (unsigned long long)float_order_key(S) << 32;  // flat index added at ranking
            } else {
              const bool moved = isnew || (c != lastp);
              n_nl[base + f] = S;
              n_k[base + f] = Kp + (isnew ? 1 : 0);
              n_tot[base + f] = totp + (moved ? 1 : 0);
              // pre-update entry with the post-update block count; slot/visits are advanced by evaluate()
              n_ov[base + f] = TabEntry{en.slot, en.blocks + (moved ? 1 : 0), en.visits, 0};
              if (isnew && Kp >= Kcap) misc[TM_ERR] = 1;
            }
          }
        }
        named_bar_sync(1, NT);
        if (misc[TM_ERR]) break;
        if (!last) {
          evaluate(base, base + count, row0 + (t0 + level - 1) % N);
          if (misc[TM_ERR]) break;
        } else {
          n_leaves = count;
        }
      }
      if (misc[TM_ERR]) { failed = true; break; }

      // ---- rank the leaves (uisrnn.py:546-552): key = (score, flat index of the index tuple)
      if (tid == 0) misc[TM_NFINITE] = 0;
      named_bar_sync(1, NT);
      if constexpr (SPILL) {
        // Leaves are enumerated in lexicographic order of their index tuples (hypothesis, c_1 .. c_L'), the order of
        // the flat index, so the leaf position breaks ties exactly as the flat index does.  It is below leaf_cap, so
        // it fits the low 32 bits at any arena size, where the flat index itself may not.
        int fin = 0;
        for (int f = tid; f < n_leaves; f += NT) {
          const unsigned skey = (unsigned)(l_key[f] >> 32);
          l_key[f] = ((unsigned long long)skey << 32) | (unsigned)f;
          fin += (skey < float_order_key(INF)) ? 1 : 0;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) fin += __shfl_xor_sync(0xffffffffu, fin, o);
        if (lane == 0 && fin) atomicAdd((int*)&misc[TM_NFINITE], fin);
      } else for (int f = tid; f < n_leaves; f += NT) {
        int chain[8];
        int lev = Lc - 1, n = (int)(l_pc[f] >> 8);
        chain[Lc - 1] = (int)(l_pc[f] & 255u);
        while (lev >= 1) { chain[lev - 1] = n_c[n]; n = n_parent[n]; --lev; }
        unsigned flat = (unsigned)n;  // hypothesis index
        for (int i = 0; i < Lc; ++i) flat = flat * (unsigned)(kmax + 1 + i) + (unsigned)chain[i];
        const unsigned skey = (unsigned)(l_key[f] >> 32);
        l_key[f] = ((unsigned long long)skey << 32) | flat;
        if (skey < float_order_key(INF)) atomicAdd((int*)&misc[TM_NFINITE], 1);
      }
      named_bar_sync(1, NT);
      const int nwin = min((int)misc[TM_NFINITE], B);
      if constexpr (SPILL) {
        if (nwin > 0) tree_select_smallest<NT>(l_key, n_leaves, nwin, wins, spill_scratch, tid, lane, warp);
      } else for (int f = tid; f < n_leaves; f += NT) {
        const unsigned long long k = l_key[f];
        int rank = 0;
        for (int q = 0; q < n_leaves; ++q) rank += (l_key[q] < k) ? 1 : 0;
        if (rank < nwin) wins[rank] = f;
      }
      named_bar_sync(1, NT);
      if (nwin == 0) { failed = true; if (tid == 0) misc[TM_ERR] = 4; named_bar_sync(1, NT); break; }

      // ---- winners become level-Lc nodes and are evaluated on the chunk's last frame
      const int wbase = lvl[Lc];
      if (wbase + nwin > NI) { failed = true; if (tid == 0) misc[TM_ERR] = 3; named_bar_sync(1, NT); break; }
      if (tid < nwin) {
        const int f = wins[tid];
        const int par = (int)(l_pc[f] >> 8), c = (int)(l_pc[f] & 255u);
        int Kp, lastp, totp;
        if (Lc == 1) { Kp = mK[par]; lastp = mLast[par]; totp = mTot[par]; }
        else { Kp = n_k[par]; lastp = n_c[par]; totp = n_tot[par]; }
        const bool isnew = (c == Kp);
        const TabEntry en = isnew ? TabEntry{kInitSlot, 0, 0, 0} : lookup(Lc - 1, par, c, tab, mK);
        const bool moved = isnew || (c != lastp);
        const int n = wbase + tid;
        n_parent[n] = par; n_c[n] = c; n_nl[n] = float_from_order_key((unsigned)(l_key[f] >> 32));
        n_k[n] = Kp + (isnew ? 1 : 0); n_tot[n] = totp + (moved ? 1 : 0);
        n_ov[n] = TabEntry{en.slot, en.blocks + (moved ? 1 : 0), en.visits, 0};
        if (isnew && Kp >= Kcap) misc[TM_ERR] = 1;
      }
      named_bar_sync(1, NT);
      if (misc[TM_ERR]) { failed = true; break; }
      evaluate(wbase, wbase + nwin, row0 + (t0 + Lc - 1) % N);
      if (misc[TM_ERR]) { failed = true; break; }

      // ---- materialise the next generation
      for (int r = warp; r < nwin; r += NW) {
        // root hypothesis of winner r
        int lev = Lc, n = wbase + r;
        while (lev >= 1) { n = n_parent[n]; --lev; }
        const int b = n;
        for (int c = lane; c < mK[b]; c += 32) ntab[(size_t)r * Kcap + c] = tab[(size_t)b * Kcap + c];
        __syncwarp();
        if (lane == 0) {
          int chain_n[8];
          lev = Lc; n = wbase + r;
          while (lev >= 1) { chain_n[lev - 1] = n; n = n_parent[n]; --lev; }
          for (int i = 0; i < Lc; ++i) {  // apply the overrides in sub-step order
            const int q = chain_n[i];
            ntab[(size_t)r * Kcap + n_c[q]] = n_ov[q];
            bp_lab[(size_t)(t0 + i) * B + r] = (unsigned)n_c[q];
            if (traced && p.dbg_win && dbg_rows + r < p.trace_capacity) p.dbg_win[(dbg_rows + r) * (1 + L) + 1 + i] = n_c[q];
          }
          const int w = wbase + r;
          nK[r] = n_k[w]; nLast[r] = n_c[w]; nTot[r] = n_tot[w]; nNl[r] = n_nl[w];
          bp_par[(size_t)step * B + r] = (unsigned)b;
          if (traced && p.dbg_win && dbg_rows + r < p.trace_capacity) {
            p.dbg_win[(dbg_rows + r) * (1 + L)] = b;
            for (int i = Lc; i < L; ++i) p.dbg_win[(dbg_rows + r) * (1 + L) + 1 + i] = -1;
            p.dbg_score[dbg_rows + r] = n_nl[w];
          }
        }
      }
      if (traced && tid == 0 && p.dbg_off) p.dbg_off[step + 1] = dbg_rows + nwin;
      dbg_rows += nwin;
      if (tid == 0) { st_steps += 1; for (int r = 0; r < nwin; ++r) st_maxk = max(st_maxk, n_k[wbase + r]); }
      named_bar_sync(1, NT);
      nb = nwin;
      gen ^= 1;
    }  // beam steps

    named_bar_sync(1, NT);
    const bool ok = !(failed || misc[TM_ERR]);
    if (tid == 0) {
      const int e = misc[TM_ERR];
      p.status[u] = ok ? 0 : (e == 1) ? -4 : (e == 2 || e == 3) ? -5 : -1;
    }
    // back-track the returned hypotheses, one per thread: hypothesis j is the j-th final rank with min_speakers
    // clusters (rank 0 when none has them, j = 0) and walks its own column chain into label plane j
    for (int j = tid; j < p.n_best; j += NT) {
      const int* fK = meta + gen * 4 * B;
      const int r0 = ok ? nbest_rank(fK, nb, spk_min(p, utt), j) : -1;
      int* lab = p.labels + ((size_t)(u / p.n_utt) * p.n_best + j) * p.label_plane + row0;
      if (r0 < 0) {
        for (int i = 0; i < N; ++i) lab[i] = -1;
      } else {
        int r = r0;
        for (int s = (TN + L - 1) / L - 1; s >= 0 && (long long)s * L + L > TN - N; --s) {
          const int t0 = s * L, Lc = min(L, TN - t0);
          for (int i = Lc - 1; i >= 0; --i) {
            const int f = t0 + i;
            if (f >= TN - N) lab[f - (TN - N)] = (int)bp_lab[(size_t)f * B + r];
          }
          r = (int)bp_par[(size_t)s * B + r];
        }
      }
      // clusters of hypothesis 0, 0 for a failed utterance; an empty utterance returns no N-best hypothesis
      if (j == 0 && p.spk_out) p.spk_out[u] = ok ? fK[r0] : 0;
      if (j == 0 && p.nbest_count) p.nbest_count[u] = (ok && N > 0) ? nbest_n(fK, nb, spk_min(p, utt), p.n_best) : 0;
      nbest_store(p, u, j, N > 0 ? r0 : -1, fK, reinterpret_cast<const float*>(fK + 3 * B));
    }
    if (p.dbg_final_scores) {
      const float* fNl = reinterpret_cast<const float*>(meta + gen * 4 * B + 3 * B);
      if (tid < B) p.dbg_final_scores[(size_t)u * B + tid] = (ok && tid < nb) ? fNl[tid] : INF;
      if (tid == 0 && p.dbg_final_k) p.dbg_final_k[u] = ok ? meta[gen * 4 * B] : 0;
    }
    if (traced && ok && p.dbg_best_mean) {
      const TabEntry* ftab = tabs + (size_t)gen * B * Kcap;
      const int K0 = meta[gen * 4 * B];
      for (int c = 0; c < K0; ++c) {
        const TabEntry en = ftab[c];
        if (tid < D) p.dbg_best_mean[(size_t)c * D + tid] = pool_mean[(size_t)en.slot * D + tid];
        for (int q = tid; q < DH; q += NT) p.dbg_best_hidden[(size_t)c * DH + q] = pool_hidden[(size_t)en.slot * DH + q];
        if (tid == 0) p.dbg_best_blocks[c] = en.blocks;
      }
    }
    named_bar_sync(1, NT);
  }  // utterances

  if (tid == 0) {
    __threadfence_block();
    misc[TM_DONE] = 1;
    atomicAdd(&p.stats[0], st_cols);
    atomicAdd(&p.stats[1], st_pass);
    atomicAdd(&p.stats[2], st_cand);
    atomicAdd(&p.stats[3], st_steps);
    atomicMax(&p.stats[4], (unsigned long long)st_maxk);
  }
}

}  // namespace uis
