// Threshold counts for label-based AP without the Q x N score matrix (dirb200_index_count_ge).
//
// The reference grades a labelled dataset with sklearn's average_precision_score over a full score row per query
// (dataset.py:83-92, evaluation.py:41-43).  With s_t = fl32(exact score) of the query's positives, that AP only needs,
// per positive, c_t = the number of rows r (r != skip_row[q]) with fl32(exact_dot_warp(q, r)) >= s_t.  For every query
// and every one of its thresholds (descending) this file counts the rows of one shard that reach it:
//
//   1. prep: per query |q| and the rounding boundaries m_t = (pred32(s_t) + s_t) / 2 (exact in fp64; pred32 = next
//      fp32 value towards -inf), per shard max |row|                         (count_prep_kernel, row_norm_max_kernel)
//   2. main pass: tiled Q x N GEMM on fp64 tensor cores (mma.sync m16n8k16 .f64, native DMMA on sm_90).  fp32 tiles
//      come to shared memory by cp.async and are widened to fp64 while the fragments are built.  fp32 x fp32
//      products are exact in fp64, and the PTX ISA specifies round-to-nearest-even (.rn, the only mode) for .f64 mma,
//      so every accumulation step rounds once and any summation order is within gamma_D * sum|q_i r_i|
//      <= gamma_D |q||r| of the exact dot product, gamma_D = D u / (1 - D u), u = 2^-53.  The tensor-core score x and
//      exact_dot_warp's e are therefore within 2 gamma_D |q||r|; eps is twice that (|q| per query, max |row| per
//      shard, per call), about 1e-12 for unit rows at D = 2048 - far below the fp32 spacing of the scores.
//      Epilogue (count_ge_gemm_kernel): fl32(e) >= s holds exactly when e > m, or e = m and s has an even significand.
//        x + eps < m_t for the query's weakest boundary: the row reaches no threshold (most elements stop here);
//        otherwise t1 = first threshold with m_t1 <= x + eps (binary search);
//          m_t1 < x - eps: the row reaches t1 and every later (lower) threshold, for certain: +1 at diff[t1];
//          else: (q, row) goes to the band list.
//      The +1s are aggregated in shared memory when the 64 queries of the tile have few enough thresholds between them,
//      with global atomics otherwise.
//   3. band: each band entry is re-scored with exact_dot_warp, rounded to fp32 and compared with the thresholds
//      directly (count_band_kernel).  A query whose entries did not fit the band list is counted again exactly over all
//      rows (count_exact_kernel) - a count is never silently wrong.
//   4. prefix sum of the difference array per query -> c_t                                   (count_scan_kernel)
#include <math.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <vector>

#include "block.cuh"
#include "conv.h"
#include "dmma.cuh"
#include "exact_dot.cuh"
#include "label_count.h"

namespace dirb {
namespace {

constexpr int CG_BM = 64, CG_BN = 128, CG_BK = 32, CG_ST = 3, CG_LD = CG_BK + 4, CG_THREADS = 256;
constexpr int CG_SMEM = CG_ST * (CG_BM + CG_BN) * CG_LD * 4;
constexpr int CG_SEG = 16384;                      // u32 per-tile counters, carved from the stage buffers after the K loop
static_assert(CG_SEG * 4 <= CG_SMEM, "tile counters must fit the stage buffers");

// workspace flags: [0] max |row| (fp32 bits, rounded up), [1] error bits (1 = thresholds not finite / not descending,
// 2 = offsets not a CSR from 0 to T), [2..3] band entries appended (u64)
constexpr int F_RMAX = 0, F_ERR = 1, F_BAND = 2;

// One warp per query: |q| (fp64), m_t of its thresholds, the difference array cleared, order checked.
__global__ void count_prep_kernel(const float* __restrict__ q32, int Q, int D, const int* __restrict__ thr_off, int T,
                                  const float* __restrict__ thr, double* __restrict__ m, double* __restrict__ qn,
                                  unsigned long long* __restrict__ diff, int* __restrict__ q_over,
                                  unsigned int* __restrict__ flags) {
  const int q = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (q >= Q) return;
  const int b = thr_off[q], e = thr_off[q + 1];
  if ((q == 0 && b != 0) || (q == Q - 1 && e != T) || b < 0 || b > e || e > T) {
    if (lane == 0) atomicOr(flags + F_ERR, 2u);
    return;
  }
  double ss = 0.0;
  for (int i = lane; i < D; i += 32) {
    const double v = q32[static_cast<int64_t>(q) * D + i];
    ss += v * v;
  }
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  if (lane == 0) {
    qn[q] = sqrt(ss);
    q_over[q] = 0;
  }
  for (int t = b + lane; t < e; t += 32) {
    const float s = thr[t];
    if (isnan(s) || isinf(s) || (t + 1 < e && thr[t + 1] > s)) atomicOr(flags + F_ERR, 1u);
    m[t] = (static_cast<double>(nextafterf(s, -INFINITY)) + static_cast<double>(s)) * 0.5;
    diff[t] = 0ull;
  }
}

// One warp per row: max |row| of the shard (fp32 rounded up; non-negative floats order like their bit patterns).
__global__ void row_norm_max_kernel(const float* __restrict__ db32, int64_t N, int D, unsigned int* __restrict__ flags) {
  const int64_t r = static_cast<int64_t>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= N) return;
  double ss = 0.0;
  for (int i = lane; i < D; i += 32) {
    const double v = db32[r * D + i];
    ss += v * v;
  }
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  if (lane == 0) atomicMax(flags + F_RMAX, __float_as_uint(__double2float_ru(sqrt(ss))));
}

// Main pass.  CTA tile 64 queries x 128 rows, 8 warps of 32 x 32, K staged 32 fp32 columns at a time (3 stages).
__global__ void __launch_bounds__(CG_THREADS, 2) count_ge_gemm_kernel(
    const float* __restrict__ q32, int Q, const float* __restrict__ db32, int64_t N, int D, int64_t offset,
    const int* __restrict__ thr_off, const double* __restrict__ m, const double* __restrict__ qn,
    const int64_t* __restrict__ skip_row, double eps_fixed, double eps_scale, const unsigned int* __restrict__ flags,
    unsigned long long* __restrict__ diff, unsigned long long* __restrict__ band, unsigned long long* __restrict__ band_cnt,
    int band_cap, int* __restrict__ q_over) {
  extern __shared__ __align__(16) float smem[];
  if (flags[F_ERR]) return;                           // malformed offsets / thresholds: reported by the host check
  float* sA = smem;                                   // [CG_ST][CG_BM][CG_LD]
  float* sB = smem + CG_ST * CG_BM * CG_LD;           // [CG_ST][CG_BN][CG_LD]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t4 = lane & 3;
  const int wm = warp & 1, wn = warp >> 1;
  const int q0 = blockIdx.y * CG_BM;
  const int64_t n0 = static_cast<int64_t>(blockIdx.x) * CG_BN;

  auto load_stage = [&](int s, int k0) {
#pragma unroll
    for (int i = 0; i < (CG_BM * CG_BK / 4) / CG_THREADS; ++i) {
      const int c = tid + i * CG_THREADS, row = c >> 3, c4 = c & 7;
      const int gq = q0 + row;
      const bool ok = gq < Q;
      cp_async16(sA + (s * CG_BM + row) * CG_LD + c4 * 4, q32 + (ok ? static_cast<int64_t>(gq) * D + k0 + c4 * 4 : 0), ok);
    }
#pragma unroll
    for (int i = 0; i < (CG_BN * CG_BK / 4) / CG_THREADS; ++i) {
      const int c = tid + i * CG_THREADS, row = c >> 3, c4 = c & 7;
      const int64_t gr = n0 + row;
      const bool ok = gr < N;
      cp_async16(sB + (s * CG_BN + row) * CG_LD + c4 * 4, db32 + (ok ? gr * D + k0 + c4 * 4 : 0), ok);
    }
  };

  double acc[2][4][4];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int k = 0; k < 4; ++k) acc[i][j][k] = 0.0;

  const int nk = D / CG_BK;
#pragma unroll
  for (int s = 0; s < CG_ST - 1; ++s) {
    if (s < nk) load_stage(s, s * CG_BK);
    cp_async_commit();
  }
  for (int kt = 0; kt < nk; ++kt) {
    cp_async_wait<CG_ST - 2>();
    __syncthreads();                                  // stage kt landed; stage kt-1 is free for the prefetch below
    if (kt + CG_ST - 1 < nk) load_stage((kt + CG_ST - 1) % CG_ST, (kt + CG_ST - 1) * CG_BK);
    cp_async_commit();
    const float* a_s = sA + (kt % CG_ST) * CG_BM * CG_LD;
    const float* b_s = sB + (kt % CG_ST) * CG_BN * CG_LD;
#pragma unroll
    for (int kk = 0; kk < CG_BK; kk += 16) {
      double b[4][4];
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) {
        const float* p = b_s + (wn * 32 + nt * 8 + g) * CG_LD + kk + t4;
#pragma unroll
        for (int i = 0; i < 4; ++i) b[nt][i] = static_cast<double>(p[4 * i]);
      }
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        double a[8];
        const float* p = a_s + (wm * 32 + mt * 16 + g) * CG_LD + kk + t4;
#pragma unroll
        for (int i = 0; i < 8; ++i) a[i] = static_cast<double>(p[(i & 1) * 8 * CG_LD + (i >> 1) * 4]);
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) dmma16816(acc[mt][nt], a, b[nt]);
      }
    }
  }
  cp_async_wait<0>();
  __syncthreads();                                    // the stage buffers become the tile's counters

  // ---- epilogue
  unsigned int* cnt_s = reinterpret_cast<unsigned int*>(smem);
  const int qa = min(q0, Q), qb = min(q0 + CG_BM, Q);
  const int seg0 = thr_off[qa];
  const int seg_len = thr_off[qb] - seg0;
  const bool use_smem = seg_len <= CG_SEG;            // uniform over the CTA
  if (use_smem)
    for (int i = tid; i < seg_len; i += CG_THREADS) cnt_s[i] = 0u;
  __syncthreads();
  auto flush = [&](int t, unsigned int n) {
    if (n == 0) return;
    if (use_smem) atomicAdd(cnt_s + (t - seg0), n);
    else atomicAdd(diff + t, static_cast<unsigned long long>(n));
  };
  const double rmax = static_cast<double>(__uint_as_float(flags[F_RMAX]));
#pragma unroll
  for (int mt = 0; mt < 2; ++mt) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int q = q0 + wm * 32 + mt * 16 + g + 8 * h;
      if (q >= Q) continue;
      const int tb = thr_off[q], te = thr_off[q + 1];
      if (tb == te) continue;
      const double m_last = m[te - 1];
      const double eps = eps_fixed > 0 ? eps_fixed : eps_scale * qn[q] * rmax;
      const int64_t skip = skip_row ? skip_row[q] : -1;
      int run_t = -1;
      unsigned int run_n = 0;
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) {
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int64_t r = n0 + wn * 32 + nt * 8 + 2 * t4 + j;
          if (r >= N || r + offset == skip) continue;
          const double x = acc[mt][nt][2 * h + j];
          if (x + eps < m_last) continue;             // below the weakest boundary: reaches no threshold
          int lo = tb, hi = te - 1;                   // first t with m_t <= x + eps (exists: m_last <= x + eps)
          while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (__ldg(m + mid) > x + eps) lo = mid + 1;
            else hi = mid;
          }
          if (__ldg(m + lo) >= x - eps) {             // within eps of a boundary: decided by the exact score
            const unsigned long long pos = atomicAdd(band_cnt, 1ull);
            if (pos < static_cast<unsigned long long>(band_cap))
              band[pos] = (static_cast<unsigned long long>(q) << 32) | static_cast<unsigned long long>(r);
            else
              q_over[q] = 1;
          } else if (lo == run_t) {
            ++run_n;
          } else {
            flush(run_t, run_n);
            run_t = lo;
            run_n = 1;
          }
        }
      }
      flush(run_t, run_n);
    }
  }
  if (use_smem) {
    __syncthreads();
    for (int i = tid; i < seg_len; i += CG_THREADS)
      if (cnt_s[i]) atomicAdd(diff + seg0 + i, static_cast<unsigned long long>(cnt_s[i]));
  }
}

// first t in [b, e) with thr[t] <= f (thr descending): the highest threshold fl32 score f reaches; e if none
__device__ __forceinline__ int first_reached(const float* __restrict__ thr, int b, int e, float f) {
  while (b < e) {
    const int mid = (b + e) >> 1;
    if (thr[mid] > f) b = mid + 1;
    else e = mid;
  }
  return b;
}

// One warp per band entry: exact score, fp32 rounding, direct comparison.  Entries of overflowed queries are skipped
// (those queries are recounted over all rows).
__global__ void count_band_kernel(const float* __restrict__ q32, const float* __restrict__ db32, int D,
                                  const int* __restrict__ thr_off, const float* __restrict__ thr,
                                  const unsigned long long* __restrict__ band, const unsigned long long* __restrict__ band_cnt,
                                  int band_cap, const int* __restrict__ q_over, unsigned long long* __restrict__ diff) {
  const int lane = threadIdx.x & 31;
  const int64_t n = static_cast<int64_t>(min(*band_cnt, static_cast<unsigned long long>(band_cap)));   // 0 after an error
  const int64_t stride = static_cast<int64_t>(gridDim.x) * (blockDim.x >> 5);
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5); i < n; i += stride) {
    const unsigned long long e = band[i];
    const int q = static_cast<int>(e >> 32);
    const int64_t r = static_cast<int64_t>(e & 0xffffffffull);
    if (q_over[q]) continue;
    const float f = __double2float_rn(exact_dot_warp(q32 + static_cast<int64_t>(q) * D, db32 + r * D, D, lane));
    if (lane == 0) {
      const int te = thr_off[q + 1];
      const int t = first_reached(thr, thr_off[q], te, f);
      if (t < te) atomicAdd(diff + t, 1ull);
    }
  }
}

// Queries whose band entries overflowed: difference array cleared, then every row scored exactly (one query per
// blockIdx.y; the clear is a separate launch so that it precedes every block's additions).
__global__ void count_clear_kernel(const int* __restrict__ q_list, int n, const int* __restrict__ thr_off,
                                   unsigned long long* __restrict__ diff) {
  const int i = blockIdx.x;
  if (i >= n) return;
  const int q = q_list[i];
  for (int t = thr_off[q] + threadIdx.x; t < thr_off[q + 1]; t += blockDim.x) diff[t] = 0ull;
}
__global__ void count_exact_kernel(const float* __restrict__ q32, const float* __restrict__ db32, int64_t N, int D,
                                   int64_t offset, const int* __restrict__ q_list, const int* __restrict__ thr_off,
                                   const float* __restrict__ thr, const int64_t* __restrict__ skip_row,
                                   unsigned long long* __restrict__ diff) {
  const int q = q_list[blockIdx.y];
  const int lane = threadIdx.x & 31;
  const int tb = thr_off[q], te = thr_off[q + 1];
  const int64_t skip = skip_row ? skip_row[q] : -1;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * (blockDim.x >> 5);
  for (int64_t r = static_cast<int64_t>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5); r < N; r += stride) {
    if (r + offset == skip) continue;
    const float f = __double2float_rn(exact_dot_warp(q32 + static_cast<int64_t>(q) * D, db32 + r * D, D, lane));
    if (lane == 0) {
      const int t = first_reached(thr, tb, te, f);
      if (t < te) atomicAdd(diff + t, 1ull);
    }
  }
}

// One warp per query: inclusive prefix sum of its difference array, in place.
__global__ void count_scan_kernel(int Q, const int* __restrict__ thr_off, unsigned long long* __restrict__ c) {
  const int q = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (q >= Q) return;
  unsigned long long carry = 0;
  for (int b = thr_off[q]; b < thr_off[q + 1]; b += 32) {
    const int t = b + lane;
    const bool in = t < thr_off[q + 1];
    const unsigned long long v = warp_scan(in ? c[t] : 0ull) + carry;
    if (in) c[t] = v;
    carry = __shfl_sync(0xffffffffu, v, 31);
  }
}

struct CountGeWs {
  double* m;
  double* qn;
  unsigned int* flags;          // 32 bytes: the F_* words, the band counter among them
  unsigned long long* band;
  int* q_over;
  int* q_list;
  size_t total;
};
CountGeWs count_ge_ws(void* base, int Q, int T, int band_cap) {
  Carver c(base);
  CountGeWs w;
  w.m = c.take<double>(T);
  w.qn = c.take<double>(Q);
  w.flags = c.take<unsigned int>(8);
  w.band = c.take<unsigned long long>(band_cap);
  w.q_over = c.take<int>(Q);
  w.q_list = c.take<int>(Q);
  w.total = c.used;
  return w;
}

}  // namespace

size_t count_ge_ws_bytes(int Q, int T, int band_cap) { return count_ge_ws(nullptr, Q, T, band_cap).total; }

int count_ge_run(const CountGeArgs& a, void* ws, CountGeStats* st, cudaStream_t stream) {
  const int Q = a.Q, T = a.T, D = a.D;
  const int64_t N = a.N;
  const CountGeWs w = count_ge_ws(ws, Q, T, a.band_cap);
  unsigned long long* band_cnt = reinterpret_cast<unsigned long long*>(w.flags + F_BAND);
  unsigned long long* diff = reinterpret_cast<unsigned long long*>(a.count);
  *st = CountGeStats{};

  DIRB_CUDA(cudaMemsetAsync(w.flags, 0, 32, stream));
  count_prep_kernel<<<static_cast<unsigned>(ceil_div(Q, 8)), 256, 0, stream>>>(a.q32, Q, D, a.thr_off, T, a.thr, w.m, w.qn,
                                                                               diff, w.q_over, w.flags);
  count_launch();
  if (N > 0) {
    row_norm_max_kernel<<<static_cast<unsigned>(ceil_div(N, 8)), 256, 0, stream>>>(a.db32, N, D, w.flags);
    count_launch();
    static std::atomic<uint64_t> attr_done{0};
    if (first_launch_on_device(attr_done))
      DIRB_CUDA(cudaFuncSetAttribute(count_ge_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, CG_SMEM));
    const double u = ldexp(1.0, -53);
    const double gamma = D * u / (1.0 - D * u);
    const dim3 grid(static_cast<unsigned>(ceil_div(N, CG_BN)), static_cast<unsigned>(ceil_div(Q, CG_BM)));
    count_ge_gemm_kernel<<<grid, CG_THREADS, CG_SMEM, stream>>>(a.q32, Q, a.db32, N, D, a.offset, a.thr_off, w.m, w.qn,
                                                                a.skip_row, a.eps, 4.0 * gamma, w.flags, diff, w.band,
                                                                band_cnt, a.band_cap, w.q_over);
    count_launch();
    count_band_kernel<<<4 * num_sms(), 256, 0, stream>>>(a.q32, a.db32, D, a.thr_off, a.thr, w.band, band_cnt, a.band_cap,
                                                         w.q_over, diff);
    count_launch();
  }
  DIRB_CUDA(cudaGetLastError());
  std::vector<int> over(Q);
  unsigned int hflags[8];
  DIRB_CUDA(cudaMemcpyAsync(over.data(), w.q_over, static_cast<size_t>(Q) * 4, cudaMemcpyDeviceToHost, stream));
  DIRB_CUDA(cudaMemcpyAsync(hflags, w.flags, 32, cudaMemcpyDeviceToHost, stream));
  DIRB_CUDA(cudaStreamSynchronize(stream));
  DIRB_REQUIRE((hflags[F_ERR] & 2u) == 0, DIRB200_EINVAL, "count_ge: threshold offsets must be a CSR running from 0 to T");
  DIRB_REQUIRE((hflags[F_ERR] & 1u) == 0, DIRB200_EINVAL,
               "count_ge: thresholds must be finite and in descending order within each query");
  unsigned long long nb;
  memcpy(&nb, hflags + F_BAND, 8);
  st->band = static_cast<int64_t>(nb);
  std::vector<int> list;
  for (int q = 0; q < Q; ++q)
    if (over[q]) list.push_back(q);
  st->fallback = static_cast<int64_t>(list.size());
  if (!list.empty()) {
    const int n = static_cast<int>(list.size());
    DIRB_CUDA(cudaMemcpyAsync(w.q_list, list.data(), static_cast<size_t>(n) * 4, cudaMemcpyHostToDevice, stream));
    count_clear_kernel<<<n, 256, 0, stream>>>(w.q_list, n, a.thr_off, diff);
    count_launch();
    const int gx = static_cast<int>(std::min<int64_t>(ceil_div(N, 8), 4 * static_cast<int64_t>(num_sms())));
    for (int i0 = 0; i0 < n; i0 += 65535) {
      const unsigned ny = static_cast<unsigned>(std::min(65535, n - i0));
      count_exact_kernel<<<dim3(gx, ny), 256, 0, stream>>>(a.q32, a.db32, N, D, a.offset, w.q_list + i0, a.thr_off, a.thr,
                                                            a.skip_row, diff);
      count_launch();
    }
  }
  count_scan_kernel<<<static_cast<unsigned>(ceil_div(Q, 8)), 256, 0, stream>>>(Q, a.thr_off, diff);
  count_launch();
  DIRB_CUDA(cudaGetLastError());
  if (!list.empty()) DIRB_CUDA(cudaStreamSynchronize(stream));    // `list` is read by the asynchronous copy above
  return 0;
}

}  // namespace dirb
