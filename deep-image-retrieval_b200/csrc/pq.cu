// Product quantisation of the inverted lists (DESIGN.md section 4.11, rules P1-P8).
//
//   pq_assign_kernel   P3 / P4: one CTA per (32 rows, sub-space m).  The rows' residuals fl32(x - c_label) of sub-space
//                      m sit in shared memory, the codebook in tiles of codewords; 8 threads per row each take every
//                      8th codeword of a tile, the fp64 distance summed over t in order with separate multiplies and
//                      adds, then the 8 minima reduce to (distance, codeword) lowest.  Training (codes m-major) and the
//                      database encoding (codes row-major) share it through the code strides.
//   pq_update_kernel   P3: one CTA per (codeword j, sub-space m): walks the training codes in row order, compacts the
//                      members of each 256-row chunk, and thread t adds column t of their residuals sequentially in
//                      fp64; then fl32(s / n), or the old codeword when n = 0.
//   pq_tables_kernel   P5: T[q][m][j] = fl32(sum_t q_{m,t} C_m[j][t]), fp64 over t in order, no FMA.
//   pq_scan_kernel     P5: one CTA per (query, group of probes): the query's table in shared memory, one thread per
//                      list row; a = fl32(e(q, c)), then a = fl32(a + T[m][code_m]) for m ascending.  Dense output in
//                      the query's segment of the block (qoff), probes in probe order.
//   pq_select_kernel   P6: one CTA per query: radix select (block_radix_kth, 8 passes of 8 bits) of the R-th largest
//                      key (a desc, row asc) over the query's segment, then the rows with a key >= it.
//   pq_refine_kernel   P7: one warp per candidate, exact_dot_warp; sort_runs_merge orders them (e desc, row asc).
#include <math.h>

#include <algorithm>

#include "block.cuh"
#include "common.h"
#include "exact_dot.cuh"

namespace dirb {
namespace {

constexpr int PQ_THREADS = 256;
constexpr int PQ_ROWS = 32;        // rows per CTA of the assignment
constexpr int PQ_LANES = 8;        // threads per row of the assignment
constexpr int PQ_MAX_SUB = 256;    // largest sub-vector (d = D / M) the kernels take
constexpr int SEL_THREADS = 1024;
constexpr int SCAN_TARGET_CTAS = 1024;   // the scan groups probes until about this many CTAs remain

// Codewords per shared-memory tile of the assignment: the whole codebook up to d = 64, beyond it the largest power of
// two whose codewords fit 64 KB.  A power of two divides 256, so the tiles cover codewords 0 .. 255 exactly.
__host__ __device__ inline int pq_tile(int d) { return d <= 64 ? 256 : d <= 128 ? 128 : 64; }
size_t pq_assign_smem(int d) { return static_cast<size_t>(PQ_ROWS + pq_tile(d)) * (d + 1) * sizeof(float); }

__global__ void __launch_bounds__(PQ_THREADS) pq_assign_kernel(const float* __restrict__ x, int64_t n, int D,
                                                               const int64_t* __restrict__ labels,
                                                               const float* __restrict__ centres,
                                                               const float* __restrict__ cb, int M,
                                                               uint8_t* __restrict__ codes, int64_t row_stride,
                                                               int64_t m_stride) {
  extern __shared__ float sm[];
  const int d = D / M, ld = d + 1, m = blockIdx.y, J = pq_tile(d);
  float* res = sm;                 // [PQ_ROWS][ld]
  float* cw = sm + PQ_ROWS * ld;   // [J][ld]
  const int64_t r0 = static_cast<int64_t>(blockIdx.x) * PQ_ROWS;
  for (int i = threadIdx.x; i < PQ_ROWS * d; i += PQ_THREADS) {
    const int r = i / d, t = i - r * d;
    const int64_t row = r0 + r;
    float v = 0.f;
    if (row < n) v = __fsub_rn(x[row * D + m * d + t], centres[labels[row] * D + m * d + t]);
    res[r * ld + t] = v;
  }
  const int r = threadIdx.x / PQ_LANES, lane = threadIdx.x % PQ_LANES;
  const float* rr = res + r * ld;
  const float* cbm = cb + static_cast<int64_t>(m) * 256 * d;
  double best = INFINITY;
  int bj = 0;
  for (int j0 = 0; j0 < 256; j0 += J) {
    __syncthreads();
    for (int i = threadIdx.x; i < J * d; i += PQ_THREADS) {
      const int j = i / d, t = i - j * d;
      cw[j * ld + t] = cbm[static_cast<int64_t>(j0 + j) * d + t];
    }
    __syncthreads();
    for (int j = lane; j < J; j += PQ_LANES) {
      const float* cc = cw + j * ld;
      double s = 0.0;
      for (int t = 0; t < d; ++t) {
        const double u = __dsub_rn(static_cast<double>(rr[t]), static_cast<double>(cc[t]));
        s = __dadd_rn(s, __dmul_rn(u, u));
      }
      if (s < best) {            // codewords ascending per thread: a tie keeps the smaller one
        best = s;
        bj = j0 + j;
      }
    }
  }
  for (int o = PQ_LANES / 2; o > 0; o >>= 1) {
    const double ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
    if (ob < best || (ob == best && oj < bj)) {
      best = ob;
      bj = oj;
    }
  }
  const int64_t row = r0 + r;
  if (lane == 0 && row < n) codes[row * row_stride + m * m_stride] = static_cast<uint8_t>(bj);
}

// codes m-major: codes[m * n + row].
__global__ void __launch_bounds__(PQ_THREADS) pq_update_kernel(const float* __restrict__ x, int64_t n, int D,
                                                               const int64_t* __restrict__ labels,
                                                               const float* __restrict__ centres,
                                                               const uint8_t* __restrict__ codes, int M,
                                                               float* __restrict__ cb,
                                                               unsigned long long* __restrict__ empty) {
  __shared__ int list[PQ_THREADS];
  __shared__ int wcnt[PQ_THREADS / 32];
  const int j = blockIdx.x, m = blockIdx.y, d = D / M;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int col = m * d + threadIdx.x;
  double s = 0.0;
  int64_t cnt = 0;
  for (int64_t c0 = 0; c0 < n; c0 += PQ_THREADS) {
    const int64_t i = c0 + threadIdx.x;
    const bool hit = i < n && codes[m * n + i] == j;
    const unsigned b = __ballot_sync(0xffffffffu, hit);
    if (lane == 0) wcnt[warp] = __popc(b);
    __syncthreads();
    int before = 0, tot = 0;
    for (int w = 0; w < PQ_THREADS / 32; ++w) {
      before += w < warp ? wcnt[w] : 0;
      tot += wcnt[w];
    }
    if (hit) list[before + __popc(b & ((1u << lane) - 1u))] = threadIdx.x;
    __syncthreads();
    if (threadIdx.x < d)
      for (int e = 0; e < tot; ++e) {
        const int64_t row = c0 + list[e];
        s = __dadd_rn(s, static_cast<double>(__fsub_rn(x[row * D + col], centres[labels[row] * D + col])));
      }
    cnt += tot;
    __syncthreads();
  }
  if (cnt == 0) {
    if (threadIdx.x == 0) atomicAdd(empty, 1ull);
    return;
  }
  if (threadIdx.x < d)
    cb[(static_cast<int64_t>(m) * 256 + j) * d + threadIdx.x] = __double2float_rn(__ddiv_rn(s, static_cast<double>(cnt)));
}

constexpr int TAB_Q = 8;   // queries per CTA of the table kernel

__global__ void __launch_bounds__(PQ_THREADS) pq_tables_kernel(const float* __restrict__ q, int Q, int D,
                                                               const float* __restrict__ cb, int M,
                                                               float* __restrict__ T) {
  __shared__ float qs[TAB_Q][PQ_MAX_SUB];
  const int m = blockIdx.x, q0 = blockIdx.y * TAB_Q, d = D / M, j = threadIdx.x;
  for (int i = threadIdx.x; i < TAB_Q * d; i += PQ_THREADS) {
    const int qi = i / d, t = i - qi * d;
    qs[qi][t] = q0 + qi < Q ? q[static_cast<int64_t>(q0 + qi) * D + m * d + t] : 0.f;
  }
  __syncthreads();
  double acc[TAB_Q];
#pragma unroll
  for (int qi = 0; qi < TAB_Q; ++qi) acc[qi] = 0.0;
  const float* c = cb + (static_cast<int64_t>(m) * 256 + j) * d;
  for (int t = 0; t < d; ++t) {
    const double cv = static_cast<double>(__ldg(c + t));
#pragma unroll
    for (int qi = 0; qi < TAB_Q; ++qi) acc[qi] = __dadd_rn(acc[qi], __dmul_rn(static_cast<double>(qs[qi][t]), cv));
  }
#pragma unroll
  for (int qi = 0; qi < TAB_Q; ++qi)
    if (q0 + qi < Q) T[(static_cast<int64_t>(q0 + qi) * M + m) * 256 + j] = __double2float_rn(acc[qi]);
}

__global__ void __launch_bounds__(PQ_THREADS) pq_scan_kernel(const float* __restrict__ T, int M,
                                                             const int64_t* __restrict__ probes,
                                                             const double* __restrict__ psc, int nprobe, int G,
                                                             const uint8_t* __restrict__ codes,
                                                             const int64_t* __restrict__ perm,
                                                             const int64_t* __restrict__ loff,
                                                             const int64_t* __restrict__ qoff, float* __restrict__ a,
                                                             int* __restrict__ arow) {
  extern __shared__ float tab[];   // [M][256]
  __shared__ int64_t s_pos;
  const int q = blockIdx.y, p0 = blockIdx.x * G, p1 = min(p0 + G, nprobe);
  const float4* src = reinterpret_cast<const float4*>(T + static_cast<int64_t>(q) * M * 256);
  for (int i = threadIdx.x; i < M * 64; i += PQ_THREADS) reinterpret_cast<float4*>(tab)[i] = src[i];
  const int64_t* pr = probes + static_cast<int64_t>(q) * nprobe;
  if (threadIdx.x == 0) {
    int64_t pos = qoff[q];
    for (int p = 0; p < p0; ++p) pos += loff[pr[p] + 1] - loff[pr[p]];
    s_pos = pos;
  }
  __syncthreads();
  int64_t pos = s_pos;
  for (int p = p0; p < p1; ++p) {
    const int64_t c = pr[p], b = loff[c], len = loff[c + 1] - b;
    const float base = __double2float_rn(psc[static_cast<int64_t>(q) * nprobe + p]);
    for (int64_t i = threadIdx.x; i < len; i += PQ_THREADS) {
      const uint2* cd = reinterpret_cast<const uint2*>(codes + (b + i) * M);
      float s = base;
      for (int m0 = 0; m0 < M; m0 += 8) {
        const uint2 v = __ldg(cd + m0 / 8);
#pragma unroll
        for (int e = 0; e < 4; ++e) s = __fadd_rn(s, tab[(m0 + e) * 256 + ((v.x >> (8 * e)) & 255u)]);
#pragma unroll
        for (int e = 0; e < 4; ++e) s = __fadd_rn(s, tab[(m0 + 4 + e) * 256 + ((v.y >> (8 * e)) & 255u)]);
      }
      a[pos + i] = s;
      arow[pos + i] = static_cast<int>(perm[b + i]);
    }
    pos += len;
  }
}

// (a desc, row asc) as one unsigned key, larger = earlier; -0 and +0 are the same score.
__device__ __forceinline__ uint64_t adc_key(float a, int row) {
  return (static_cast<uint64_t>(f2key(a == 0.f ? 0.f : a)) << 32) | static_cast<uint32_t>(0x7fffffff - row);
}

__global__ void __launch_bounds__(SEL_THREADS) pq_select_kernel(const float* __restrict__ a, const int* __restrict__ arow,
                                                                const int64_t* __restrict__ qoff, int R, int cap2,
                                                                int* __restrict__ rows, int* __restrict__ cnt) {
  __shared__ uint32_t hist[256], bc[2];
  __shared__ int s_slot;
  const int q = blockIdx.x;
  const int64_t b = qoff[q], n = qoff[q + 1] - b;
  int* out = rows + static_cast<int64_t>(q) * cap2;
  if (threadIdx.x == 0) s_slot = 0;
  __syncthreads();
  // the R-th largest key: keys are distinct, so exactly R rows reach it
  const uint64_t thr =
      n > R ? block_radix_kth<uint64_t>([&](int64_t i) { return adc_key(a[b + i], arow[b + i]); }, n, R, hist, bc) : 0;
  for (int64_t i = threadIdx.x; i < n; i += SEL_THREADS)
    if (n <= R || adc_key(a[b + i], arow[b + i]) >= thr) out[atomicAdd(&s_slot, 1)] = arow[b + i];
  __syncthreads();
  if (threadIdx.x == 0) cnt[q] = s_slot;
}

__global__ void __launch_bounds__(PQ_THREADS) pq_refine_kernel(const float* __restrict__ q32, int D,
                                                               const float* __restrict__ x, const int* __restrict__ rows,
                                                               const int* __restrict__ cnt, int cap2,
                                                               double* __restrict__ sc) {
  const int q = blockIdx.y, lane = threadIdx.x & 31;
  const int i = blockIdx.x * (PQ_THREADS / 32) + (threadIdx.x >> 5);
  if (i >= cnt[q]) return;
  const int64_t o = static_cast<int64_t>(q) * cap2 + i;
  const double e = exact_dot_warp(q32 + static_cast<int64_t>(q) * D, x + static_cast<int64_t>(rows[o]) * D, D, lane);
  if (lane == 0) sc[o] = e;
}

// dirb200_pq_search: the ADC scores and rows of the block's probed rows, then the candidates in sort_runs_merge's layout.
struct PqSearchWs {
  float* a;
  int* arow;
  int* cnt;
  unsigned long long* status;
  SortScratch s;
  size_t total;
};
PqSearchWs pq_search_ws(void* base, int Q, int64_t total, int R) {
  Carver c(base);
  PqSearchWs w;
  w.a = c.take<float>(static_cast<size_t>(std::max<int64_t>(total, 1)));
  w.arow = c.take<int>(static_cast<size_t>(std::max<int64_t>(total, 1)));
  w.cnt = c.take<int>(Q);
  w.status = c.take<unsigned long long>(8);
  w.s = take_sort_scratch(c, Q, sort_run_cap(R));
  w.total = c.used;
  return w;
}

bool pq_shape_ok(int D, int M) {
  return (M == 8 || M == 16 || M == 32 || M == 64 || M == 128) && D > 0 && D % 64 == 0 && D % M == 0 &&
         D / M <= PQ_MAX_SUB;
}

// The device address of rows that are device memory or pinned host memory; null for pageable host memory.
const float* device_rows(const float* rows) {
  cudaPointerAttributes at{};
  if (cudaPointerGetAttributes(&at, rows) != cudaSuccess) {
    cudaGetLastError();
    return nullptr;
  }
  if (at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged) return rows;
  if (at.type == cudaMemoryTypeHost) return static_cast<const float*>(at.devicePointer);
  return nullptr;
}

}  // namespace
}  // namespace dirb

using namespace dirb;

extern "C" {

int dirb200_pq_assign(const float* x_dev, int64_t n, int D, const int64_t* labels_dev, const float* centres_dev,
                      const float* codebooks_dev, int M, uint8_t* codes_dev, int m_major, void* stream_) {
  DIRB_REQUIRE(n >= 1 && x_dev && labels_dev && centres_dev && codebooks_dev && codes_dev, DIRB200_EINVAL,
               "bad arguments");
  DIRB_REQUIRE(pq_shape_ok(D, M), DIRB200_ENOTSUP, "unsupported PQ shape (D %d, M %d)", D, M);
  DIRB_REQUIRE(n <= (int64_t(1) << 31) * PQ_ROWS, DIRB200_ENOTSUP, "too many rows");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  static std::atomic<uint64_t> once{0};
  if (first_launch_on_device(once))
    DIRB_CUDA(cudaFuncSetAttribute(pq_assign_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   static_cast<int>(pq_assign_smem(PQ_MAX_SUB))));
  const int d = D / M;
  pq_assign_kernel<<<dim3(static_cast<unsigned>(ceil_div(n, PQ_ROWS)), M), PQ_THREADS, pq_assign_smem(d), stream>>>(
      x_dev, n, D, labels_dev, centres_dev, codebooks_dev, M, codes_dev, m_major ? 1 : M, m_major ? n : 1);
  count_launch();
  DIRB_CUDA(cudaGetLastError());
  return 0;
}

int dirb200_pq_update(const float* x_dev, int64_t n, int D, const int64_t* labels_dev, const float* centres_dev,
                      const uint8_t* codes_dev, int M, float* codebooks_dev, int64_t* empty_dev, void* stream_) {
  DIRB_REQUIRE(n >= 1 && x_dev && labels_dev && centres_dev && codes_dev && codebooks_dev && empty_dev, DIRB200_EINVAL,
               "bad arguments");
  DIRB_REQUIRE(pq_shape_ok(D, M), DIRB200_ENOTSUP, "unsupported PQ shape (D %d, M %d)", D, M);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DIRB_CUDA(cudaMemsetAsync(empty_dev, 0, 8, stream));
  pq_update_kernel<<<dim3(256, M), PQ_THREADS, 0, stream>>>(x_dev, n, D, labels_dev, centres_dev, codes_dev, M,
                                                            codebooks_dev,
                                                            reinterpret_cast<unsigned long long*>(empty_dev));
  count_launch();
  DIRB_CUDA(cudaGetLastError());
  return 0;
}

int dirb200_pq_tables(const float* q_dev, int Q, int D, const float* codebooks_dev, int M, float* tables_dev,
                      void* stream_) {
  DIRB_REQUIRE(Q >= 1 && q_dev && codebooks_dev && tables_dev, DIRB200_EINVAL, "bad arguments");
  DIRB_REQUIRE(pq_shape_ok(D, M), DIRB200_ENOTSUP, "unsupported PQ shape (D %d, M %d)", D, M);
  DIRB_REQUIRE(Q <= 65535 * TAB_Q, DIRB200_ENOTSUP, "too many queries (%d)", Q);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  pq_tables_kernel<<<dim3(M, static_cast<unsigned>(ceil_div(Q, TAB_Q))), PQ_THREADS, 0, stream>>>(q_dev, Q, D,
                                                                                                 codebooks_dev, M,
                                                                                                 tables_dev);
  count_launch();
  DIRB_CUDA(cudaGetLastError());
  return 0;
}

size_t dirb200_pq_search_ws_bytes(int Q, int64_t total, int R) {
  if (Q < 1 || total < 0 || R < 1) return 0;
  return pq_search_ws(nullptr, Q, total, R).total;
}

int dirb200_pq_search(const float* q_dev, int Q, int D, const float* tables_dev, int M, const int64_t* probes_dev,
                      const double* probe_scores_dev, int nprobe, const uint8_t* codes_dev, const int64_t* perm_dev,
                      const int64_t* list_off_dev, const int64_t* qoff_dev, int64_t total, const float* rows, int R,
                      int k, void* ws_dev, double* out_scores, int64_t* out_rows, double* ms, void* stream_) {
  DIRB_REQUIRE(Q >= 1 && Q <= 65535 && nprobe >= 1 && total >= 0 && R >= 1 && k >= 1 && k <= R && q_dev &&
                   tables_dev && probes_dev && probe_scores_dev && codes_dev && perm_dev && list_off_dev && qoff_dev &&
                   rows && ws_dev && out_scores && out_rows,
               DIRB200_EINVAL, "bad arguments");
  DIRB_REQUIRE(pq_shape_ok(D, M), DIRB200_ENOTSUP, "unsupported PQ shape (D %d, M %d)", D, M);
  const float* x = device_rows(rows);
  DIRB_REQUIRE(x, DIRB200_EINVAL, "rows must be device memory or pinned host memory (the device cannot read pageable "
               "host memory)");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const PqSearchWs w = pq_search_ws(ws_dev, Q, total, R);
  const int cap2 = sort_run_cap(R);
  cudaEvent_t ev[4] = {};
  if (ms)
    for (auto& e : ev) DIRB_CUDA(cudaEventCreate(&e));
  if (ms) DIRB_CUDA(cudaEventRecord(ev[0], stream));
  static std::atomic<uint64_t> once{0};
  const size_t tab_smem = static_cast<size_t>(M) * 256 * sizeof(float);
  if (first_launch_on_device(once))
    DIRB_CUDA(cudaFuncSetAttribute(pq_scan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 128 * 256 * 4));
  const int G = static_cast<int>(std::clamp<int64_t>(static_cast<int64_t>(Q) * nprobe / SCAN_TARGET_CTAS, 1, nprobe));
  pq_scan_kernel<<<dim3(static_cast<unsigned>(ceil_div(nprobe, G)), Q), PQ_THREADS, tab_smem, stream>>>(
      tables_dev, M, probes_dev, probe_scores_dev, nprobe, G, codes_dev, perm_dev, list_off_dev, qoff_dev, w.a, w.arow);
  if (ms) DIRB_CUDA(cudaEventRecord(ev[1], stream));
  pq_select_kernel<<<Q, SEL_THREADS, 0, stream>>>(w.a, w.arow, qoff_dev, R, cap2, w.s.rows, w.cnt);
  if (ms) DIRB_CUDA(cudaEventRecord(ev[2], stream));
  pq_refine_kernel<<<dim3(static_cast<unsigned>(ceil_div(R, PQ_THREADS / 32)), Q), PQ_THREADS, 0, stream>>>(
      q_dev, D, x, w.s.rows, w.cnt, cap2, w.s.sc);
  count_launch(3);
  DIRB_TRY(sort_runs_merge(w.s.rows, w.cnt, cap2, w.s.sc, w.s.run_ix, Q, k, 0, w.status, out_scores, out_rows, stream));
  if (ms) {
    DIRB_CUDA(cudaEventRecord(ev[3], stream));
    DIRB_CUDA(cudaEventSynchronize(ev[3]));
    for (int i = 0; i < 3; ++i) {
      float t = 0.f;
      DIRB_CUDA(cudaEventElapsedTime(&t, ev[i], ev[i + 1]));
      ms[i] = t;
    }
    for (auto& e : ev) cudaEventDestroy(e);
  }
  DIRB_CUDA(cudaGetLastError());
  return 0;
}

}  // extern "C"
