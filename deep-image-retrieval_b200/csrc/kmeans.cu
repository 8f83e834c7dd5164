// Spherical k-means on unit fp32 rows (DESIGN.md section 4.9, rules K4-K7).  The assignment itself (rules K2 / K3) is
// dirb200_index_nearest over the centres (search.cu); this file holds what happens around it.
//
//   km_stats_kernel       per row: cluster sizes (which the update's offsets reuse), labels that differ from the previous
//                         assignment, and the objective in int64 fixed point (each score in units of 2^-32, rounded to
//                         nearest).  Integer sums: the same result whatever order the atomics take.
//   km_empty_kernel       the number of empty clusters.
//   km_relocate_kernel    K4: rows ordered by (score asc, row asc) with sort_runs_merge (key -score); one thread gives each
//                         empty cluster, ascending, the next row in that order whose cluster still has >= 2 rows.  A row
//                         passed over never qualifies later (donor sizes only shrink, a filled cluster holds 1 row), so
//                         one pointer walks the order once.
//   km_sum_kernel         K5: rows ordered by (label, row) with sort_runs_merge (key -label); one block per (cluster, 256
//                         columns) sums the cluster's rows in chunks of 256, each chunk sequentially, the chunk sums in
//                         chunk order, in fp64.
//   km_norm_kernel        K5: one block per cluster: ||s||^2 (thread t sums the columns t, t + 256, ... in order, then a
//                         halving tree over the 256 threads) and the centre fl32(s / sqrt(||s||^2)); s = 0 keeps the old
//                         centre.
//   km_pp_*_kernel        K7: per draw one launch over the rows (exact score with the newest centre, best score, weight
//                         in units of 2^-32, per-block weight sums) and one single-block launch that finds the drawn row
//                         from the prefix sums.  No host round trip between draws.
#include <math.h>

#include <algorithm>

#include "block.cuh"
#include "common.h"
#include "exact_dot.cuh"

namespace dirb {
namespace {

constexpr int KM_THREADS = 256;
constexpr int KM_SCAN = 1024;
constexpr int KM_CHUNK = 256;      // rows per chunk of the centre sums (rule K5)
constexpr int KM_COLS = 256;       // columns per block of the centre sums
constexpr int PP_ROWS = 256;       // rows per block of a k-means++ weight launch
constexpr double FIX32 = 4294967296.0;

unsigned grid_for(int64_t n) { return static_cast<unsigned>(std::max<int64_t>(1, std::min<int64_t>(ceil_div(n, KM_THREADS), 8192))); }

// acc[0] = labels that differ from prev (every row when prev is null), acc[1] = sum of rint(score * 2^32).
__global__ void km_stats_kernel(const int64_t* __restrict__ labels, const double* __restrict__ scores,
                                const int64_t* __restrict__ prev, int64_t n, int* __restrict__ counts,
                                unsigned long long* __restrict__ acc) {
  long long changed = 0, obj = 0;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t l = labels[i];
    atomicAdd(counts + l, 1);
    changed += (prev == nullptr || prev[i] != l) ? 1 : 0;
    obj += __double2ll_rn(scores[i] * FIX32);
  }
  for (int o = 16; o > 0; o >>= 1) {
    changed += __shfl_down_sync(0xffffffffu, changed, o);
    obj += __shfl_down_sync(0xffffffffu, obj, o);
  }
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(acc, static_cast<unsigned long long>(changed));
    atomicAdd(acc + 1, static_cast<unsigned long long>(obj));
  }
}

__global__ void km_empty_kernel(const int* __restrict__ counts, int k, unsigned long long* __restrict__ acc) {
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < k; c += gridDim.x * blockDim.x)
    if (counts[c] == 0) atomicAdd(acc, 1ull);
}

// Sort input of sort_runs_merge: rows 0 .. n-1 with key -label (label asc, row asc) or -score (score asc, row asc).
__global__ void km_keys_kernel(const int64_t* __restrict__ labels, const double* __restrict__ scores, int64_t n,
                               int* __restrict__ rows, double* __restrict__ key) {
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    rows[i] = static_cast<int>(i);
    key[i] = labels ? -static_cast<double>(labels[i]) : -scores[i];
  }
}

// off[c] = rows of clusters < c (exclusive scan of the sizes), off[k] = n.
__global__ void __launch_bounds__(KM_SCAN) km_offsets_kernel(const int* __restrict__ counts, int k, int64_t* __restrict__ off) {
  __shared__ long long warp_sums[KM_SCAN / 32];
  long long carry = 0;
  for (int base = 0; base < k; base += KM_SCAN) {
    const int c = base + threadIdx.x;
    const long long v = c < k ? counts[c] : 0;
    long long tot;
    const long long incl = block_scan(v, warp_sums, &tot);
    if (c < k) off[c] = carry + incl - v;
    carry += tot;
  }
  if (threadIdx.x == 0) off[k] = carry;
}

__global__ void __launch_bounds__(KM_SCAN) km_relocate_kernel(const int64_t* __restrict__ order, int64_t n, int k,
                                                              int64_t* __restrict__ labels, int* __restrict__ counts,
                                                              long long* __restrict__ moves) {
  __shared__ int empty[KM_SCAN];
  __shared__ int warp_cnt[KM_SCAN / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int64_t next = 0;
  long long mv = 0;
  for (int base = 0; base < k; base += KM_SCAN) {
    const int c = base + threadIdx.x;
    const bool e = c < k && counts[c] == 0;
    const unsigned bal = __ballot_sync(0xffffffffu, e);
    if (lane == 0) warp_cnt[warp] = __popc(bal);
    __syncthreads();
    if (e) {
      int before = 0;
      for (int w = 0; w < warp; ++w) before += warp_cnt[w];
      empty[before + __popc(bal & ((1u << lane) - 1u))] = c;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      int ne = 0;
      for (int w = 0; w < KM_SCAN / 32; ++w) ne += warp_cnt[w];
      for (int j = 0; j < ne; ++j) {
        while (next < n) {
          const int64_t r = order[next++];
          const int64_t l = labels[r];
          if (counts[l] >= 2) {
            counts[l] -= 1;
            labels[r] = empty[j];
            counts[empty[j]] = 1;
            ++mv;
            break;
          }
        }
      }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) *moves = mv;
}

// s[c][col] for the columns of block y: chunks of KM_CHUNK members summed sequentially, chunk sums added in order.
__global__ void __launch_bounds__(KM_COLS) km_sum_kernel(const float* __restrict__ x, int d,
                                                         const int64_t* __restrict__ members,
                                                         const int64_t* __restrict__ off, double* __restrict__ s) {
  const int c = blockIdx.x;
  const int col = blockIdx.y * KM_COLS + threadIdx.x;
  if (col >= d) return;
  const int64_t b = off[c], e = off[c + 1];
  double tot = 0.0;
  for (int64_t c0 = b; c0 < e; c0 += KM_CHUNK) {
    const int64_t c1 = min(c0 + KM_CHUNK, e);
    double acc = 0.0;
#pragma unroll 8
    for (int64_t p = c0; p < c1; ++p) acc += static_cast<double>(__ldg(x + __ldg(members + p) * d + col));
    tot += acc;
  }
  s[static_cast<int64_t>(c) * d + col] = tot;
}

__global__ void __launch_bounds__(KM_THREADS) km_norm_kernel(const double* __restrict__ s, int d,
                                                             float* __restrict__ centres,
                                                             unsigned long long* __restrict__ zero_sums) {
  __shared__ double red[KM_THREADS];
  const double* sc = s + static_cast<int64_t>(blockIdx.x) * d;
  double v = 0.0;
  for (int j = threadIdx.x; j < d; j += KM_THREADS) v = __dadd_rn(v, __dmul_rn(sc[j], sc[j]));
  red[threadIdx.x] = v;
  __syncthreads();
  for (int st = KM_THREADS / 2; st > 0; st >>= 1) {
    if (threadIdx.x < st) red[threadIdx.x] = __dadd_rn(red[threadIdx.x], red[threadIdx.x + st]);
    __syncthreads();
  }
  const double ss = red[0];
  if (ss == 0.0) {
    if (threadIdx.x == 0) atomicAdd(zero_sums, 1ull);
    return;
  }
  const double nrm = __dsqrt_rn(ss);
  float* out = centres + static_cast<int64_t>(blockIdx.x) * d;
  for (int j = threadIdx.x; j < d; j += KM_THREADS) out[j] = __double2float_rn(__ddiv_rn(sc[j], nrm));
}

__global__ void km_pp_start_kernel(int64_t first, int64_t* __restrict__ chosen, uint8_t* __restrict__ flag) {
  chosen[0] = first;
  flag[first] = 1;
}

// Draw j >= 1: best[i] = max over the chosen centres of e(x_i, x_c); w[i] = 0 for chosen rows, else
// rint(max(0, 2 - 2 best[i]) * 2^32); bsum[block] = the block's weight sum.
__global__ void __launch_bounds__(KM_THREADS) km_pp_weight_kernel(const float* __restrict__ x, int64_t n, int d,
                                                                  const int64_t* __restrict__ chosen, int j,
                                                                  double* __restrict__ best,
                                                                  const uint8_t* __restrict__ flag,
                                                                  long long* __restrict__ w, long long* __restrict__ bsum) {
  __shared__ long long sh[PP_ROWS];
  const int64_t c = chosen[j - 1];
  if (c < 0) return;                          // an earlier draw found no weight left: nothing more is drawn
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t base = static_cast<int64_t>(blockIdx.x) * PP_ROWS;
  const float* xc = x + c * d;
  for (int r = warp; r < PP_ROWS; r += KM_THREADS / 32) {
    const int64_t i = base + r;
    long long wi = 0;
    if (i < n) {
      const double e = exact_dot_warp(x + i * d, xc, d, lane);
      const double b = j == 1 ? e : fmax(best[i], e);
      wi = flag[i] ? 0 : __double2ll_rn(fmax(0.0, 2.0 - 2.0 * b) * FIX32);
      if (lane == 0) {
        best[i] = b;
        w[i] = wi;
      }
    }
    if (lane == 0) sh[r] = wi;
  }
  __syncthreads();
  for (int st = PP_ROWS / 2; st > 0; st >>= 1) {
    if (threadIdx.x < st) sh[threadIdx.x] += sh[threadIdx.x + st];
    __syncthreads();
  }
  if (threadIdx.x == 0) bsum[blockIdx.x] = sh[0];
}

// Draw j: T = sum of the weights, t = min(floor(u_j * double(T)), T - 1); the drawn row is the first whose inclusive
// weight prefix exceeds t (the block from the block sums, then the row inside it).  T = 0 draws -1.
__global__ void __launch_bounds__(KM_SCAN) km_pp_select_kernel(const long long* __restrict__ bsum, int64_t nb,
                                                               const long long* __restrict__ w, int64_t n,
                                                               const double* __restrict__ u, int j,
                                                               int64_t* __restrict__ chosen, uint8_t* __restrict__ flag) {
  __shared__ long long warp_sums[KM_SCAN / 32];
  __shared__ long long s_before;
  __shared__ int64_t s_blk;
  if (chosen[j - 1] < 0) {
    if (threadIdx.x == 0) chosen[j] = -1;
    return;
  }
  long long part = 0;
  for (int64_t b = threadIdx.x; b < nb; b += KM_SCAN) part += bsum[b];
  long long T;
  block_scan(part, warp_sums, &T);
  if (T == 0) {
    if (threadIdx.x == 0) chosen[j] = -1;
    return;
  }
  long long t = static_cast<long long>(floor(u[j - 1] * static_cast<double>(T)));
  if (t > T - 1) t = T - 1;
  long long carry = 0;
  for (int64_t base = 0; base < nb; base += KM_SCAN) {
    const int64_t b = base + threadIdx.x;
    const long long v = b < nb ? bsum[b] : 0;
    long long tot;
    const long long incl = carry + block_scan(v, warp_sums, &tot);
    if (b < nb && incl > t && incl - v <= t) {
      s_blk = b;
      s_before = incl - v;
    }
    carry += tot;
  }
  __syncthreads();
  const int64_t i = s_blk * PP_ROWS + threadIdx.x;
  const long long v = (threadIdx.x < PP_ROWS && i < n) ? w[i] : 0;
  long long tot;
  const long long incl = s_before + block_scan(v, warp_sums, &tot);
  if (v > 0 && incl > t && incl - v <= t) {
    chosen[j] = i;
    flag[i] = 1;
  }
}

struct SortWs {
  SortScratch s;
  double* out_key;
  int64_t* order;
  int* cnt;
  unsigned long long* status;
};
// The sort buffers of n rows, taken from c.
SortWs sort_ws(Carver& c, int64_t n) {
  SortWs w;
  w.s = take_sort_scratch(c, 1, sort_run_cap(std::max<int64_t>(n, 1)));
  w.out_key = c.take<double>(n);
  w.order = c.take<int64_t>(n);
  w.cnt = c.take<int>(1);
  w.status = c.take<unsigned long long>(8);
  return w;
}

// Rows 0 .. n-1 into w.order by (label asc, row asc) when labels is given, else by (score asc, row asc).
int order_rows(const SortWs& w, const int64_t* labels, const double* scores, int64_t n, cudaStream_t stream) {
  const int n32 = static_cast<int>(n);
  km_keys_kernel<<<grid_for(n), KM_THREADS, 0, stream>>>(labels, scores, n, w.s.rows, w.s.sc);
  count_launch();
  DIRB_CUDA(cudaMemcpyAsync(w.cnt, &n32, 4, cudaMemcpyHostToDevice, stream));
  return sort_runs_merge(w.s.rows, w.cnt, sort_run_cap(n), w.s.sc, w.s.run_ix, 1, n32, 0, w.status, w.out_key, w.order,
                         stream);
}

// dirb200_kmeans_relocate: the moves counter, then the sort buffers
struct RelocateWs {
  long long* moves;
  SortWs sort;
  size_t total;
};
RelocateWs relocate_ws(void* base, int64_t n) {
  Carver c(base);
  RelocateWs w;
  w.moves = c.take<long long>(1);
  w.sort = sort_ws(c, n);
  w.total = c.used;
  return w;
}

struct UpdateWs {
  int64_t* off;
  double* s;
  unsigned long long* zero;
  SortWs sort;
  size_t total;
};
UpdateWs update_ws(void* base, int64_t n, int k, int d) {
  Carver c(base);
  UpdateWs w;
  w.off = c.take<int64_t>(static_cast<size_t>(k) + 1);
  w.s = c.take<double>(static_cast<size_t>(k) * d);
  w.zero = c.take<unsigned long long>(1);
  w.sort = sort_ws(c, n);
  w.total = c.used;
  return w;
}

struct PpWs {
  double* best;
  long long* w;
  long long* bsum;
  double* u;
  uint8_t* flag;
  size_t total;
};
PpWs pp_ws(void* base, int64_t n, int k) {
  Carver c(base);
  PpWs w;
  w.best = c.take<double>(n);
  w.w = c.take<long long>(n);
  w.bsum = c.take<long long>(ceil_div(n, PP_ROWS));
  w.u = c.take<double>(k);
  w.flag = c.take<uint8_t>(n);
  w.total = c.used;
  return w;
}

constexpr int64_t KM_MAX_ROWS = int64_t(1) << 29;    // k-means++ weights: up to 2^34 units each, an int64 total

}  // namespace
}  // namespace dirb

using namespace dirb;

extern "C" {

size_t dirb200_kmeans_stats_workspace_bytes(int64_t n, int k) {
  (void)n;
  (void)k;
  return 256;
}

int dirb200_kmeans_stats(const int64_t* labels_dev, const double* scores_dev, const int64_t* prev_dev, int64_t n, int k,
                         void* ws_dev, int* counts_dev, int64_t out[3], void* stream_) {
  DIRB_REQUIRE(n >= 1 && k >= 1 && labels_dev && scores_dev && ws_dev && counts_dev && out, DIRB200_EINVAL,
               "bad arguments");
  DIRB_REQUIRE(n < KM_MAX_ROWS, DIRB200_ENOTSUP, "too many rows (%lld)", static_cast<long long>(n));
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  unsigned long long* acc = static_cast<unsigned long long*>(ws_dev);
  DIRB_CUDA(cudaMemsetAsync(acc, 0, 24, stream));
  DIRB_CUDA(cudaMemsetAsync(counts_dev, 0, static_cast<size_t>(k) * 4, stream));
  km_stats_kernel<<<grid_for(n), KM_THREADS, 0, stream>>>(labels_dev, scores_dev, prev_dev, n, counts_dev, acc);
  km_empty_kernel<<<grid_for(k), KM_THREADS, 0, stream>>>(counts_dev, k, acc + 2);
  count_launch(2);
  DIRB_CUDA(cudaMemcpyAsync(out, acc, 24, cudaMemcpyDeviceToHost, stream));
  DIRB_CUDA(cudaStreamSynchronize(stream));
  DIRB_CUDA(cudaGetLastError());
  return 0;
}

size_t dirb200_kmeans_relocate_workspace_bytes(int64_t n) {
  if (n < 1) return 0;
  return relocate_ws(nullptr, n).total;
}

int dirb200_kmeans_relocate(int64_t* labels_dev, const double* scores_dev, int64_t n, int k, int* counts_dev,
                            void* ws_dev, int64_t* moves_out, void* stream_) {
  DIRB_REQUIRE(n >= 1 && k >= 1 && k <= n && labels_dev && scores_dev && counts_dev && ws_dev && moves_out,
               DIRB200_EINVAL, "bad arguments");
  DIRB_REQUIRE(n < KM_MAX_ROWS, DIRB200_ENOTSUP, "too many rows (%lld)", static_cast<long long>(n));
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const RelocateWs w = relocate_ws(ws_dev, n);
  DIRB_TRY(order_rows(w.sort, nullptr, scores_dev, n, stream));
  km_relocate_kernel<<<1, KM_SCAN, 0, stream>>>(w.sort.order, n, k, labels_dev, counts_dev, w.moves);
  count_launch();
  long long mv = 0;
  DIRB_CUDA(cudaMemcpyAsync(&mv, w.moves, 8, cudaMemcpyDeviceToHost, stream));
  DIRB_CUDA(cudaStreamSynchronize(stream));
  DIRB_CUDA(cudaGetLastError());
  *moves_out = mv;
  return 0;
}

size_t dirb200_kmeans_update_workspace_bytes(int64_t n, int k, int d) {
  if (n < 1 || k < 1 || d < 1) return 0;
  return update_ws(nullptr, n, k, d).total;
}

int dirb200_kmeans_update(const float* x32_dev, int64_t n, int d, const int64_t* labels_dev, const int* counts_dev, int k,
                          float* centres_dev, void* ws_dev, int64_t* zero_sums_out, void* stream_) {
  DIRB_REQUIRE(n >= 1 && k >= 1 && x32_dev && labels_dev && counts_dev && centres_dev && ws_dev && zero_sums_out,
               DIRB200_EINVAL, "bad arguments");
  DIRB_REQUIRE(d > 0 && d % 64 == 0, DIRB200_ENOTSUP, "descriptor dim must be a multiple of 64 (got %d)", d);
  DIRB_REQUIRE(n < KM_MAX_ROWS, DIRB200_ENOTSUP, "too many rows (%lld)", static_cast<long long>(n));
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const UpdateWs w = update_ws(ws_dev, n, k, d);
  DIRB_CUDA(cudaMemsetAsync(w.zero, 0, 8, stream));
  km_offsets_kernel<<<1, KM_SCAN, 0, stream>>>(counts_dev, k, w.off);
  count_launch();
  DIRB_TRY(order_rows(w.sort, labels_dev, nullptr, n, stream));
  km_sum_kernel<<<dim3(static_cast<unsigned>(k), static_cast<unsigned>(ceil_div(d, KM_COLS))), KM_COLS, 0, stream>>>(
      x32_dev, d, w.sort.order, w.off, w.s);
  km_norm_kernel<<<static_cast<unsigned>(k), KM_THREADS, 0, stream>>>(w.s, d, centres_dev, w.zero);
  count_launch(2);
  unsigned long long z = 0;
  DIRB_CUDA(cudaMemcpyAsync(&z, w.zero, 8, cudaMemcpyDeviceToHost, stream));
  DIRB_CUDA(cudaStreamSynchronize(stream));
  DIRB_CUDA(cudaGetLastError());
  *zero_sums_out = static_cast<int64_t>(z);
  return 0;
}

size_t dirb200_kmeans_pp_workspace_bytes(int64_t n, int k) {
  if (n < 1 || k < 1) return 0;
  return pp_ws(nullptr, n, k).total;
}

int dirb200_kmeans_pp(const float* x32_dev, int64_t n, int d, int64_t first, const double* u_host, int k, void* ws_dev,
                      int64_t* chosen_dev, void* stream_) {
  DIRB_REQUIRE(n >= 1 && k >= 1 && k <= n && first >= 0 && first < n && x32_dev && ws_dev && chosen_dev &&
                   (k == 1 || u_host),
               DIRB200_EINVAL, "bad arguments");
  DIRB_REQUIRE(d > 0 && d % 64 == 0, DIRB200_ENOTSUP, "descriptor dim must be a multiple of 64 (got %d)", d);
  DIRB_REQUIRE(n < KM_MAX_ROWS, DIRB200_ENOTSUP, "too many rows (%lld): the weight total would overflow int64",
               static_cast<long long>(n));
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const PpWs w = pp_ws(ws_dev, n, k);
  const int64_t nb = ceil_div(n, PP_ROWS);
  DIRB_CUDA(cudaMemsetAsync(w.flag, 0, static_cast<size_t>(n), stream));
  if (k > 1) DIRB_CUDA(cudaMemcpyAsync(w.u, u_host, static_cast<size_t>(k - 1) * 8, cudaMemcpyHostToDevice, stream));
  km_pp_start_kernel<<<1, 1, 0, stream>>>(first, chosen_dev, w.flag);
  count_launch();
  for (int j = 1; j < k; ++j) {
    km_pp_weight_kernel<<<static_cast<unsigned>(nb), KM_THREADS, 0, stream>>>(x32_dev, n, d, chosen_dev, j, w.best, w.flag,
                                                                             w.w, w.bsum);
    km_pp_select_kernel<<<1, KM_SCAN, 0, stream>>>(w.bsum, nb, w.w, n, w.u, j, chosen_dev, w.flag);
    count_launch(2);
  }
  DIRB_CUDA(cudaStreamSynchronize(stream));
  DIRB_CUDA(cudaGetLastError());
  return 0;
}

}  // extern "C"
