// The chain plan of a score call made on the device (uis_score_device_ids in include/uisrnn_b200.h): arbitrary int64
// ids per frame in, canonical labels and the plan plan_chains (uis_api.cu) makes out, with nothing read back.
//
//   1. sort the (id, frame) pairs stably by id, then stably by utterance: every run of equal ids in an utterance is one
//      chain, its frames in frame order, its head the id's first appearance
//   2. flag the heads at their frames; an exclusive scan of the flags in frame order gives, at a head, its chain id
//      (chains of earlier utterances + clusters of its utterance opened before it): the utterance base subtracted, the
//      canonical label, which every frame of the run takes
//   3. the run length is the chain length; a stable descending sort of the chain ids by length gives the queue order
//      (ties in (utterance, canonical label) order, as std::stable_sort in plan_chains), a scan of the sorted lengths
//      chain_off, and each frame goes to chain_off[rank of its chain] + its place in the run
//   4. chains, queued (length >= 2: a prefix of the order) and max_k land in counts[3]
// The index arrays are int32 (rows < 2^31); chain_off / chain_rows are the chain kernel's long long arrays.
#include <cub/cub.cuh>

#include "uis_launch.cuh"

namespace uis {
namespace {

constexpr int kPlanBlock = 256;

struct MaxOp {
  __device__ __forceinline__ int operator()(int a, int b) const { return a > b ? a : b; }
};

// The scratch arrays of one plan, carved from one workspace.
struct PlanWs {
  long long* id_sorted;  // [rows]     ids after the first sort (not read: CUB needs the key output)
  int *utt, *iota, *frame_a, *utt_key, *utt_sorted, *srow, *first, *excl, *headpos, *runstart, *len, *len_sorted,
      *cid_sorted, *rank;
  void* temp;
  size_t temp_bytes;
  size_t total;
};

int bits_for(long long v) {  // bits of the largest key value v (at least 1)
  int b = 1;
  while (b < 62 && (1ll << b) <= v) ++b;
  return b;
}

size_t cub_temp_bytes(long long rows, int U) {
  const int n = (int)rows;
  size_t worst = 0, b = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, b, (const long long*)nullptr, (long long*)nullptr, (const int*)nullptr,
                                  (int*)nullptr, n);
  worst = std::max(worst, b);
  cub::DeviceRadixSort::SortPairs(nullptr, b, (const int*)nullptr, (int*)nullptr, (const int*)nullptr, (int*)nullptr, n,
                                  0, bits_for(U));
  worst = std::max(worst, b);
  cub::DeviceRadixSort::SortPairsDescending(nullptr, b, (const int*)nullptr, (int*)nullptr, (const int*)nullptr,
                                            (int*)nullptr, n, 0, bits_for(rows));
  worst = std::max(worst, b);
  cub::DeviceScan::ExclusiveSum(nullptr, b, (const int*)nullptr, (int*)nullptr, n + 1);
  worst = std::max(worst, b);
  cub::DeviceScan::InclusiveScan(nullptr, b, (const int*)nullptr, (int*)nullptr, MaxOp{}, n);
  worst = std::max(worst, b);
  cub::DeviceScan::ExclusiveSum(nullptr, b, (const int*)nullptr, (long long*)nullptr, n + 1);
  worst = std::max(worst, b);
  return worst;
}

PlanWs carve(void* base, long long rows, int U) {
  PlanWs w{};
  size_t at = 0;
  auto take = [&](size_t bytes) {
    char* p = static_cast<char*>(base) + at;
    at += (bytes + 255) / 256 * 256;
    return p;
  };
  const size_t n = (size_t)rows, n1 = n + 1;
  w.id_sorted = reinterpret_cast<long long*>(take(n * 8));
  int** arrays[] = {&w.utt, &w.iota, &w.frame_a, &w.utt_key, &w.utt_sorted, &w.srow, &w.headpos, &w.runstart, &w.len,
                    &w.cid_sorted, &w.rank};
  for (int** a : arrays) *a = reinterpret_cast<int*>(take(n * 4));
  w.first = reinterpret_cast<int*>(take(n1 * 4));
  w.excl = reinterpret_cast<int*>(take(n1 * 4));
  w.len_sorted = reinterpret_cast<int*>(take(n1 * 4));
  w.temp_bytes = base ? 0 : cub_temp_bytes(rows, U);
  w.temp = take(w.temp_bytes);
  w.total = at;
  return w;
}

#define GRID_STRIDE(i, n) for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < (n); \
                               i += (long long)gridDim.x * blockDim.x)

// utt[r]: the utterance of frame r (the last u with row_off[u] <= r: empty utterances are skipped); iota[r] = r
__global__ void plan_rows_kernel(const long long* __restrict__ row_off, int U, long long rows, int* utt, int* iota) {
  GRID_STRIDE(r, rows) {
    int lo = 0, hi = U;
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (row_off[mid] <= r) lo = mid; else hi = mid;
    }
    utt[r] = lo;
    iota[r] = (int)r;
  }
}

__global__ void plan_gather_kernel(const int* __restrict__ utt, const int* __restrict__ frame, long long rows, int* key) {
  GRID_STRIDE(i, rows) key[i] = utt[frame[i]];
}

// first[r] = 1 at the first frame of every (utterance, id); headpos[i] = i at a run's first sorted position, else 0
__global__ void plan_heads_kernel(const long long* __restrict__ ids, const int* __restrict__ srow,
                                  const int* __restrict__ su, long long rows, int* first, int* headpos) {
  GRID_STRIDE(i, rows) {
    const int r = srow[i];
    const bool head = i == 0 || su[i] != su[i - 1] || ids[r] != ids[srow[i - 1]];
    first[r] = head ? 1 : 0;
    headpos[i] = head ? (int)i : 0;
  }
}

// canonical labels of every frame; the length of every chain, by chain id, at the run's last position
__global__ void plan_runs_kernel(const int* __restrict__ srow, const int* __restrict__ su, const int* __restrict__ runstart,
                                 const int* __restrict__ excl, const long long* __restrict__ row_off, long long rows,
                                 int* labels, int* labels_out, int* len) {
  GRID_STRIDE(i, rows) {
    const int s = runstart[i];
    const int cid = excl[srow[s]];
    const int canon = cid - excl[row_off[su[i]]];
    const int r = srow[i];
    labels[r] = canon;
    if (labels_out) labels_out[r] = canon;
    if (i + 1 == rows || runstart[i + 1] == i + 1) len[cid] = (int)(i - s + 1);
  }
}

// rank[chain id] = its place in the queue; counts[0] = chains, counts[1] = queued (the sorted lengths descend, so
// each count is where its threshold is crossed)
__global__ void plan_rank_kernel(const int* __restrict__ len_sorted, const int* __restrict__ cid_sorted, long long rows,
                                 int* rank, int* counts) {
  GRID_STRIDE(k, rows) {
    const int n = len_sorted[k], next = k + 1 < rows ? len_sorted[k + 1] : 0;
    if (n > 0) rank[cid_sorted[k]] = (int)k;
    if (n >= 1 && next < 1) counts[0] = (int)(k + 1);
    if (n >= 2 && next < 2) counts[1] = (int)(k + 1);
  }
}

__global__ void plan_scatter_kernel(const int* __restrict__ srow, const int* __restrict__ runstart,
                                    const int* __restrict__ excl, const int* __restrict__ rank,
                                    const long long* __restrict__ chain_off, long long rows, long long* chain_rows) {
  GRID_STRIDE(i, rows) {
    const int s = runstart[i];
    const int k = rank[excl[srow[s]]];
    chain_rows[chain_off[k] + (i - s)] = srow[i];
  }
}

// counts[2] = the most clusters in one utterance
__global__ void plan_max_k_kernel(const int* __restrict__ excl, const long long* __restrict__ row_off, int U, int* counts) {
  GRID_STRIDE(u, U) {
    const int k = excl[row_off[u + 1]] - excl[row_off[u]];
    if (k > 0) atomicMax(counts + 2, k);
  }
}

}  // namespace

size_t score_plan_bytes(long long rows, int U) { return carve(nullptr, rows, U).total; }

#define PLAN_CU(call)                         \
  do {                                        \
    const cudaError_t e_ = (call);            \
    if (e_ != cudaSuccess) return e_;         \
  } while (0)

cudaError_t score_plan(const long long* ids, const long long* row_off, int U, long long rows, void* ws, size_t ws_bytes,
                       int* labels, int* labels_out, long long* chain_off, long long* chain_rows, int* counts,
                       int num_sms, cudaStream_t st) {
  PlanWs w = carve(ws, rows, U);
  w.temp_bytes = ws_bytes - (size_t)(static_cast<char*>(w.temp) - static_cast<char*>(ws));
  const int n = (int)rows;
  const unsigned grid = (unsigned)std::max<long long>(1, std::min<long long>((rows + kPlanBlock - 1) / kPlanBlock,
                                                                             (long long)num_sms * 16));
  PLAN_CU(cudaMemsetAsync(counts, 0, 3 * sizeof(int), st));
  PLAN_CU(cudaMemsetAsync(w.first + rows, 0, sizeof(int), st));
  PLAN_CU(cudaMemsetAsync(w.len, 0, (size_t)rows * sizeof(int), st));
  PLAN_CU(cudaMemsetAsync(w.len_sorted + rows, 0, sizeof(int), st));
  plan_rows_kernel<<<grid, kPlanBlock, 0, st>>>(row_off, U, rows, w.utt, w.iota);
  PLAN_CU(cudaGetLastError());
  // 1. stable by id (all 64 bits), then stable by utterance
  PLAN_CU(cub::DeviceRadixSort::SortPairs(w.temp, w.temp_bytes, ids, w.id_sorted, w.iota, w.frame_a, n, 0, 64, st));
  plan_gather_kernel<<<grid, kPlanBlock, 0, st>>>(w.utt, w.frame_a, rows, w.utt_key);
  PLAN_CU(cudaGetLastError());
  PLAN_CU(cub::DeviceRadixSort::SortPairs(w.temp, w.temp_bytes, w.utt_key, w.utt_sorted, w.frame_a, w.srow, n, 0,
                                          bits_for(U), st));
  // 2. heads, their chain ids (frame order) and each position's run start
  plan_heads_kernel<<<grid, kPlanBlock, 0, st>>>(ids, w.srow, w.utt_sorted, rows, w.first, w.headpos);
  PLAN_CU(cudaGetLastError());
  PLAN_CU(cub::DeviceScan::ExclusiveSum(w.temp, w.temp_bytes, w.first, w.excl, n + 1, st));
  PLAN_CU(cub::DeviceScan::InclusiveScan(w.temp, w.temp_bytes, w.headpos, w.runstart, MaxOp{}, n, st));
  plan_runs_kernel<<<grid, kPlanBlock, 0, st>>>(w.srow, w.utt_sorted, w.runstart, w.excl, row_off, rows, labels,
                                                labels_out, w.len);
  PLAN_CU(cudaGetLastError());
  // 3. the queue: chain ids by descending length (unused ids have length 0 and sort last), offsets, rows
  PLAN_CU(cub::DeviceRadixSort::SortPairsDescending(w.temp, w.temp_bytes, w.len, w.len_sorted, w.iota, w.cid_sorted, n,
                                                    0, bits_for(rows), st));
  plan_rank_kernel<<<grid, kPlanBlock, 0, st>>>(w.len_sorted, w.cid_sorted, rows, w.rank, counts);
  PLAN_CU(cudaGetLastError());
  PLAN_CU(cub::DeviceScan::ExclusiveSum(w.temp, w.temp_bytes, w.len_sorted, chain_off, n + 1, st));
  plan_scatter_kernel<<<grid, kPlanBlock, 0, st>>>(w.srow, w.runstart, w.excl, w.rank, chain_off, rows, chain_rows);
  PLAN_CU(cudaGetLastError());
  // 4. max_k
  plan_max_k_kernel<<<(unsigned)std::max(1, std::min((U + kPlanBlock - 1) / kPlanBlock, num_sms * 16)), kPlanBlock, 0,
                      st>>>(w.excl, row_off, U, counts);
  return cudaGetLastError();
}

}  // namespace uis
