// Truncated diffusion (Iscen et al. CVPR 2017): each query is solved on the mutual-kNN subgraph of its own top-m rows
// instead of the whole database graph (dirb200_diffusion_trunc_*).  DESIGN.md section 4.7, rules T1-T6.
//
//   trunc_build_kernel   one block per query: R_q (the first m list entries) sorted by global index, carrying each
//                        row's list position; every local row walks its global CSR row of A in ascending j and keeps
//                        the j found in R_q (binary search) -> local columns and A values, ascending; d'_i summed in
//                        that order from 0, u'_i = 1/sqrt(d'_i) (0 if d'_i = 0), S'_ij = A_ij * (u'_i * u'_j); seeds
//                        y' = max(s, 0)^gamma at the first kq list entries.  The expressions of fill_kernel,
//                        normalize_kernel and seeds_kernel (diffusion.cu).
//   trunc_cg_kernel      one block per query, all iterations in one launch: the full solver's arithmetic and its
//                        reduction order (fixed 64-row blocks, warp slot w taking rows w, w + 8, ... in order, the 8
//                        slots added in order, the block partials by cg_scalar_kernel's 256-thread tree), so with
//                        m >= N the solution is dirb200_diffusion_solve's bit for bit.  The vectors f, r, p, Ap live in
//                        shared memory when 32 m bytes fit, else in a per-query slice of the workspace.
//   trunc_gather_kernel + sort_runs_merge + trunc_emit_kernel: the local rows ordered by (f' desc, row asc), then the
//                        plain exact list past m'.
//   trunc_rank_kernel    per target: inside R_q or not (binary search), f', and the R_q rows ranking before it.
// No atomics on values anywhere: a given input gives the same bits on every run, whatever the query block.
#include <limits.h>
#include <math.h>

#include <algorithm>

#include "block.cuh"
#include "common.h"

namespace dirb {
namespace {

constexpr int TB_THREADS = 256;
constexpr int TS_THREADS = 256;             // = cg_scalar_kernel's tree width
constexpr int RB = 64;                      // rows per reduction block, as in the full solver
constexpr int CG_WARPS = 8;
constexpr int SMEM_OPT_IN = 227 * 1024;     // dynamic shared memory a block of an H100 may opt into
constexpr int KEY_SMEM_MAX = 128 * 1024;    // sort keys of R_q in shared memory up to 16384 rows

int pow2_at_least(int m) { int P = 1; while (P < m) P <<= 1; return P; }
bool keys_in_smem(int m) { return size_t(pow2_at_least(m)) * 8 <= size_t(KEY_SMEM_MAX); }
size_t cg_smem_bytes(int m) { return size_t(m) * 4 * 8; }
bool cg_in_smem(int m) { return cg_smem_bytes(m) + TS_THREADS * 8 + 1024 <= size_t(SMEM_OPT_IN); }

__device__ __forceinline__ int key_row(uint64_t key) { return static_cast<int>(key >> 32); }

// ------------------------------------------------------------------------------------------------ local subgraph
// seeds_kernel's expression at the first kq entries of each list, parked in dd [Q][m] in list order until
// trunc_build_kernel moves them to their local rows
__global__ void trunc_seed_kernel(const double* __restrict__ list_score, int Q, int m, int kq, double gamma,
                                  double* __restrict__ dd) {
  const int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= static_cast<int64_t>(Q) * kq) return;
  const int64_t o = (t / kq) * m + t % kq;
  dd[o] = pow(fmax(list_score[o], 0.0), gamma);
}

// key[l] = (global row << 32) | list position, sorted ascending: local row l is the l-th row of R_q by index.
// ELL storage column-major per query: entry e of local row l at [q][e][l] (coalesced over rows).
template <bool kShared>
__global__ void __launch_bounds__(TB_THREADS, 1) trunc_build_kernel(
    const int64_t* __restrict__ row_ptr, const int* __restrict__ col, const double* __restrict__ a, int kw,
    const int64_t* __restrict__ list_idx, int m, int kq, uint64_t* __restrict__ key_ws, int64_t* __restrict__ rows, int* __restrict__ lcnt, int* __restrict__ lcol,
    double* __restrict__ lval, double* __restrict__ dd, double* __restrict__ uu, double* __restrict__ y) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int q = blockIdx.x;
  int P = 1;
  while (P < m) P <<= 1;
  uint64_t* key = kShared ? reinterpret_cast<uint64_t*>(smem) : key_ws + static_cast<int64_t>(q) * P;
  const int64_t qm = static_cast<int64_t>(q) * m;
  for (int e = threadIdx.x; e < P; e += TB_THREADS)
    key[e] = e < m ? (static_cast<uint64_t>(list_idx[qm + e]) << 32) | static_cast<uint32_t>(e) : ~0ull;
  __syncthreads();
  block_bitonic_sort<TB_THREADS>(key, P, [](uint64_t a, uint64_t b) { return a < b; });
  for (int l = threadIdx.x; l < m; l += TB_THREADS) {       // the seeds to their local rows, before dd is reused
    const int pos = static_cast<int>(key[l] & 0xffffffffu);
    y[qm + l] = pos < kq ? dd[qm + pos] : 0.0;
  }
  __syncthreads();
  int* lc = lcol + qm * kw;
  double* lv = lval + qm * kw;
  for (int l = threadIdx.x; l < m; l += TB_THREADS) {
    const uint64_t kl = key[l];
    const int g = key_row(kl);
    rows[qm + l] = g;
    int c = 0;
    double d = 0.0;
    const int64_t e1 = row_ptr[g + 1];
    for (int64_t e = row_ptr[g]; e < e1; ++e) {
      const int j = col[e];
      int lo = 0, hi = m;
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (key_row(key[mid]) < j) lo = mid + 1; else hi = mid;
      }
      if (lo < m && key_row(key[lo]) == j) {
        const double v = a[e];
        lc[static_cast<int64_t>(c) * m + l] = lo;
        lv[static_cast<int64_t>(c) * m + l] = v;
        d += v;
        ++c;
      }
    }
    lcnt[qm + l] = c;
    dd[qm + l] = d;
    uu[qm + l] = d > 0.0 ? 1.0 / sqrt(d) : 0.0;
  }
  __syncthreads();
  for (int l = threadIdx.x; l < m; l += TB_THREADS) {
    const double ui = uu[qm + l];
    const int c = lcnt[qm + l];
    for (int e = 0; e < c; ++e) {
      const int64_t o = static_cast<int64_t>(e) * m + l;
      lv[o] = lv[o] * (ui * uu[qm + lc[o]]);
    }
  }
}

// ------------------------------------------------------------------------------------------------ fused CG
// x . z over m rows in the full solver's order: block b of 64 rows, slot w sums rows w, w + 8, ... in order, the slots
// are added in order (block_partial); thread t adds the blocks t, t + 256, ... from 0 and the 256 sums go through
// cg_scalar_kernel's tree.  Every thread returns the total.
__device__ __forceinline__ double ordered_dot(const double* x, const double* z, int m, double* red) {
  const int nb = (m + RB - 1) / RB;
  double v = 0.0;
  for (int b0 = 0; b0 < nb; b0 += TS_THREADS) {
    const int b = b0 + threadIdx.x;
    if (b >= nb) break;
    double s = 0.0;
#pragma unroll
    for (int w = 0; w < CG_WARPS; ++w) {
      double acc = 0.0;
#pragma unroll
      for (int i = w; i < RB; i += CG_WARPS) {
        const int row = b * RB + i;
        if (row < m) acc += x[row] * z[row];
      }
      s = w == 0 ? acc : s + acc;
    }
    v += s;
  }
  red[threadIdx.x] = v;
  __syncthreads();
  for (int h = TS_THREADS / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h) red[threadIdx.x] += red[threadIdx.x + h];
    __syncthreads();
  }
  const double t = red[0];
  __syncthreads();
  return t;
}

template <bool kShared>
__global__ void __launch_bounds__(TS_THREADS) trunc_cg_kernel(
    const int* __restrict__ lcnt, const int* __restrict__ lcol, const double* __restrict__ lval, int kw,
    const double* __restrict__ y, int m, double alpha, int iters, double tol, double* __restrict__ vec_ws,
    double* __restrict__ f_out, int* __restrict__ iters_out, double* __restrict__ resid_out) {
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ double red[TS_THREADS];
  const int q = blockIdx.x;
  const int64_t qm = static_cast<int64_t>(q) * m;
  double* base = kShared ? reinterpret_cast<double*>(smem) : vec_ws + qm * 4;
  double* f = base;
  double* r = base + m;
  double* p = base + 2 * static_cast<int64_t>(m);
  double* ap = base + 3 * static_cast<int64_t>(m);
  const int* cnt = lcnt + qm;
  const int* lc = lcol + qm * kw;
  const double* lv = lval + qm * kw;
  for (int i = threadIdx.x; i < m; i += TS_THREADS) {
    const double v = y[qm + i];
    f[i] = 0.0;
    r[i] = v;
    p[i] = v;
  }
  __syncthreads();
  // the scalars of cg_scalar_kernel, kept by thread 0 in shared memory (few registers live across the division and
  // square-root subroutines)
  __shared__ double s_yy, s_rr, s_al, s_be, s_res;
  __shared__ int s_done, s_act;
  {
    const double t = ordered_dot(r, r, m, red);
    if (threadIdx.x == 0) {
      s_yy = t;
      s_rr = t;
      s_done = 0;
      s_res = sqrt(t);
      s_act = t > 0.0 && !(sqrt(t) <= tol * sqrt(t));
    }
    __syncthreads();
  }
  for (int it = 0; it < iters && s_act; ++it) {
    for (int i = threadIdx.x; i < m; i += TS_THREADS) {      // ap = p - a S p, nonzeros in ascending column order
      double sp = 0.0;
      const int c = cnt[i];
      for (int e = 0; e < c; ++e) {
        const int64_t o = static_cast<int64_t>(e) * m + i;
        const double v = lv[o];
        sp += v * p[lc[o]];
      }
      const double pi = p[i];
      const double api = pi - alpha * sp;
      ap[i] = api;
    }
    __syncthreads();
    const double pap = ordered_dot(p, ap, m, red);
    if (threadIdx.x == 0) s_al = s_rr / pap;
    __syncthreads();
    const double al = s_al;
    for (int i = threadIdx.x; i < m; i += TS_THREADS) {
      f[i] = f[i] + al * p[i];
      const double rv = r[i] - al * ap[i];
      r[i] = rv;
    }
    __syncthreads();
    const double t = ordered_dot(r, r, m, red);
    if (threadIdx.x == 0) {
      s_be = t / s_rr;
      s_rr = t;
      s_done += 1;
      s_res = sqrt(t);
      if (sqrt(t) <= tol * sqrt(s_yy)) s_act = 0;
    }
    __syncthreads();
    if (it + 1 < iters && s_act) {
      const double be = s_be;
      for (int i = threadIdx.x; i < m; i += TS_THREADS) p[i] = r[i] + be * p[i];
      __syncthreads();
    }
  }
  for (int i = threadIdx.x; i < m; i += TS_THREADS) f_out[qm + i] = f[i];
  if (threadIdx.x == 0) {
    iters_out[q] = s_done;
    resid_out[q] = s_res;
  }
}

// ------------------------------------------------------------------------------------------------ ranking
// grid (row chunks, Q): the m local (row, f') pairs of each query -> sort_runs_merge's candidate layout
__global__ void trunc_gather_kernel(const int64_t* __restrict__ rows, const double* __restrict__ f, int m, int cap2,
                                    int* __restrict__ rows32, double* __restrict__ sc, int* __restrict__ cnt) {
  const int q = blockIdx.y;
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l < m) {
    const int64_t o = static_cast<int64_t>(q) * cap2 + l;
    rows32[o] = static_cast<int>(rows[static_cast<int64_t>(q) * m + l]);
    sc[o] = f[static_cast<int64_t>(q) * m + l];
  }
  if (l == 0) cnt[q] = m;
}

// grid (position chunks, Q): out[q][p] = the ordered local rows for p < kk, the exact list's entry p after them
__global__ void trunc_emit_kernel(const double* __restrict__ top_s, const int64_t* __restrict__ top_i, int kk,
                                  const double* __restrict__ list_score, const int64_t* __restrict__ list_idx, int lw,
                                  int k, double* __restrict__ out_s, int64_t* __restrict__ out_i) {
  const int q = blockIdx.y;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= k) return;
  const int64_t o = static_cast<int64_t>(q) * k + p;
  if (p < kk) {
    out_s[o] = top_s[static_cast<int64_t>(q) * kk + p];
    out_i[o] = top_i[static_cast<int64_t>(q) * kk + p];
  } else {
    out_s[o] = list_score[static_cast<int64_t>(q) * lw + p];
    out_i[o] = list_idx[static_cast<int64_t>(q) * lw + p];
  }
}

// one block per query, one warp per target: inside R_q (binary search in the ascending rows), f', and for a flagged
// target inside R_q the number of R_q rows before it under rule T6 (f' desc, row asc; -0 == +0 as doubles compare)
__global__ void __launch_bounds__(256) trunc_rank_kernel(const int64_t* __restrict__ rows, const double* __restrict__ f,
                                                         int m, const int* __restrict__ t_off,
                                                         const int64_t* __restrict__ t_rows,
                                                         const uint8_t* __restrict__ t_flags,
                                                         uint8_t* __restrict__ inside, double* __restrict__ value,
                                                         int64_t* __restrict__ above) {
  const int q = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t* rq = rows + static_cast<int64_t>(q) * m;
  const double* fq = f + static_cast<int64_t>(q) * m;
  for (int a = t_off[q] + warp; a < t_off[q + 1]; a += 8) {
    const int64_t t = t_rows[a];
    int lo = 0, hi = m;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (rq[mid] < t) lo = mid + 1; else hi = mid;
    }
    const bool in = lo < m && rq[lo] == t;
    const double ft = in ? fq[lo] : 0.0;
    int c = 0;
    if (in && t_flags[a])
      for (int l = lane; l < m; l += 32) c += fq[l] > ft || (fq[l] == ft && rq[l] < t);
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if (lane == 0) {
      inside[a] = in;
      value[a] = ft;
      above[a] = c;
    }
  }
}

// ------------------------------------------------------------------------------------------------ workspaces
struct BuildWs { uint64_t* keys; size_t total; };
BuildWs build_ws(void* base, int Q, int m) {
  Carver c(base);
  BuildWs w;
  w.keys = c.take<uint64_t>(keys_in_smem(m) ? 1 : size_t(Q) * pow2_at_least(m));
  w.total = c.used;
  return w;
}

struct TopkWs { SortScratch s; int* cnt; double* top_s; int64_t* top_i; unsigned long long* status; size_t total; };
TopkWs topk_ws(void* base, int Q, int m, int k) {
  Carver c(base);
  TopkWs w;
  const size_t qk = size_t(Q) * std::min(k, m);
  w.s = take_sort_scratch(c, Q, sort_run_cap(m));
  w.cnt = c.take<int>(Q);
  w.top_s = c.take<double>(qk);
  w.top_i = c.take<int64_t>(qk);
  w.status = c.take<unsigned long long>(8);
  w.total = c.used;
  return w;
}

}  // namespace
}  // namespace dirb

using namespace dirb;

extern "C" {

size_t dirb200_diffusion_trunc_build_workspace_bytes(int Q, int m) {
  if (Q < 1 || m < 1) return 0;
  return build_ws(nullptr, Q, m).total;
}

int dirb200_diffusion_trunc_build(const int64_t* row_ptr_dev, const int* col_dev, const double* a_dev, int64_t N,
                                  int kw, const int64_t* list_idx_dev, const double* list_score_dev, int Q, int m,
                                  int kq, double gamma, void* ws_dev, int64_t* rows_dev, int* lcnt_dev, int* lcol_dev,
                                  double* lval_dev, double* d_dev, double* u_dev, double* y_dev, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DIRB_REQUIRE(N >= 1 && N < INT_MAX && Q >= 1 && m >= 1 && m <= N && kw >= 1, DIRB200_EINVAL,
               "diffusion_trunc_build: bad sizes N %lld, Q %d, m %d, kw %d", (long long)N, Q, m, kw);
  DIRB_REQUIRE(kq >= 1 && kq <= m, DIRB200_EINVAL, "diffusion_trunc_build: need 1 <= kq <= m (got kq %d, m %d)", kq, m);
  DIRB_REQUIRE(gamma > 0.0, DIRB200_EINVAL, "diffusion_trunc_build: gamma must be > 0 (got %g)", gamma);
  DIRB_REQUIRE(row_ptr_dev && col_dev && a_dev && list_idx_dev && list_score_dev && ws_dev && rows_dev && lcnt_dev &&
               lcol_dev && lval_dev && d_dev && u_dev && y_dev, DIRB200_EINVAL, "diffusion_trunc_build: null argument");
  DIRB_TRY(require_sm90());
  BuildWs w = build_ws(ws_dev, Q, m);
  trunc_seed_kernel<<<static_cast<unsigned>(ceil_div(static_cast<int64_t>(Q) * kq, 256)), 256, 0, stream>>>(
      list_score_dev, Q, m, kq, gamma, d_dev);
  if (keys_in_smem(m)) {
    const int bytes = pow2_at_least(m) * 8;
    DIRB_CUDA(cudaFuncSetAttribute(trunc_build_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    trunc_build_kernel<true><<<Q, TB_THREADS, bytes, stream>>>(row_ptr_dev, col_dev, a_dev, kw, list_idx_dev, m, kq,
                                                               w.keys, rows_dev, lcnt_dev,
                                                               lcol_dev, lval_dev, d_dev, u_dev, y_dev);
  } else {
    trunc_build_kernel<false><<<Q, TB_THREADS, 0, stream>>>(row_ptr_dev, col_dev, a_dev, kw, list_idx_dev, m, kq,
                                                            w.keys, rows_dev, lcnt_dev,
                                                            lcol_dev, lval_dev, d_dev, u_dev, y_dev);
  }
  count_launch(2);
  DIRB_CUDA(cudaGetLastError());
  return 0;
}

size_t dirb200_diffusion_trunc_solve_workspace_bytes(int Q, int m) {
  if (Q < 1 || m < 1) return 0;
  Carver c(nullptr);
  c.take<char>(cg_in_smem(m) ? 1 : size_t(Q) * cg_smem_bytes(m));
  return c.used;
}

int dirb200_diffusion_trunc_solve(const int* lcnt_dev, const int* lcol_dev, const double* lval_dev, int kw,
                                  const double* y_dev, int Q, int m, double alpha, int iters, double tol, void* ws_dev,
                                  double* f_dev, int* iters_dev, double* resid_dev, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DIRB_REQUIRE(Q >= 1 && m >= 1 && kw >= 1, DIRB200_EINVAL, "diffusion_trunc_solve: bad sizes Q %d, m %d, kw %d", Q, m,
               kw);
  DIRB_REQUIRE(alpha >= 0.0 && alpha < 1.0 && iters >= 1 && tol >= 0.0, DIRB200_EINVAL,
               "diffusion_trunc_solve: need 0 <= alpha < 1, iters >= 1, tol >= 0 (got %g, %d, %g)", alpha, iters, tol);
  DIRB_REQUIRE(lcnt_dev && lcol_dev && lval_dev && y_dev && ws_dev && f_dev && iters_dev && resid_dev, DIRB200_EINVAL,
               "diffusion_trunc_solve: null argument");
  DIRB_TRY(require_sm90());
  if (cg_in_smem(m)) {
    const int bytes = static_cast<int>(cg_smem_bytes(m));
    DIRB_CUDA(cudaFuncSetAttribute(trunc_cg_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    trunc_cg_kernel<true><<<Q, TS_THREADS, bytes, stream>>>(lcnt_dev, lcol_dev, lval_dev, kw, y_dev, m, alpha, iters,
                                                            tol, static_cast<double*>(ws_dev), f_dev, iters_dev,
                                                            resid_dev);
  } else {
    trunc_cg_kernel<false><<<Q, TS_THREADS, 0, stream>>>(lcnt_dev, lcol_dev, lval_dev, kw, y_dev, m, alpha, iters, tol,
                                                         static_cast<double*>(ws_dev), f_dev, iters_dev, resid_dev);
  }
  count_launch();
  DIRB_CUDA(cudaGetLastError());
  return 0;
}

size_t dirb200_diffusion_trunc_topk_workspace_bytes(int Q, int m, int k) {
  if (Q < 1 || m < 1 || k < 1) return 0;
  return topk_ws(nullptr, Q, m, k).total;
}

int dirb200_diffusion_trunc_topk(const int64_t* rows_dev, const double* f_dev, int Q, int m,
                                 const int64_t* list_idx_dev, const double* list_score_dev, int list_width, int k,
                                 void* ws_dev, double* scores_dev, int64_t* idx_dev, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DIRB_REQUIRE(Q >= 1 && m >= 1 && k >= 1 && m < INT_MAX, DIRB200_EINVAL,
               "diffusion_trunc_topk: bad sizes Q %d, m %d, k %d", Q, m, k);
  DIRB_REQUIRE(k <= m || (list_idx_dev && list_score_dev && list_width >= k), DIRB200_EINVAL,
               "diffusion_trunc_topk: k %d > m %d needs the exact lists to depth >= k (got %d)", k, m, list_width);
  DIRB_REQUIRE(Q <= 65535, DIRB200_ENOTSUP, "diffusion_trunc_topk: at most 65535 queries per call (got %d)", Q);
  DIRB_REQUIRE(rows_dev && f_dev && ws_dev && scores_dev && idx_dev, DIRB200_EINVAL, "diffusion_trunc_topk: null argument");
  DIRB_TRY(require_sm90());
  TopkWs w = topk_ws(ws_dev, Q, m, k);
  const int cap2 = sort_run_cap(m);
  const int kk = std::min(k, m);
  trunc_gather_kernel<<<dim3(static_cast<unsigned>(ceil_div(m, 256)), Q), 256, 0, stream>>>(rows_dev, f_dev, m, cap2,
                                                                                            w.s.rows, w.s.sc, w.cnt);
  count_launch();
  DIRB_TRY(sort_runs_merge(w.s.rows, w.cnt, cap2, w.s.sc, w.s.run_ix, Q, kk, 0, w.status, w.top_s, w.top_i, stream));
  trunc_emit_kernel<<<dim3(static_cast<unsigned>(ceil_div(k, 256)), Q), 256, 0, stream>>>(
      w.top_s, w.top_i, kk, list_score_dev, list_idx_dev, list_width, k, scores_dev, idx_dev);
  count_launch();
  DIRB_CUDA(cudaGetLastError());
  return 0;
}

int dirb200_diffusion_trunc_rank_count(const int64_t* rows_dev, const double* f_dev, int Q, int m,
                                       const int* t_off_dev, const int64_t* t_rows_dev, const uint8_t* t_flags_dev,
                                       int T, uint8_t* inside_dev, double* value_dev, int64_t* above_dev,
                                       void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DIRB_REQUIRE(Q >= 1 && m >= 1 && T >= 0, DIRB200_EINVAL, "diffusion_trunc_rank_count: bad sizes Q %d, m %d, T %d", Q,
               m, T);
  DIRB_REQUIRE(rows_dev && f_dev && t_off_dev && (T == 0 || (t_rows_dev && t_flags_dev && inside_dev && value_dev &&
               above_dev)), DIRB200_EINVAL, "diffusion_trunc_rank_count: null argument");
  DIRB_TRY(require_sm90());
  if (T == 0) return 0;
  trunc_rank_kernel<<<Q, 256, 0, stream>>>(rows_dev, f_dev, m, t_off_dev, t_rows_dev, t_flags_dev, inside_dev,
                                           value_dev, above_dev);
  count_launch();
  DIRB_CUDA(cudaGetLastError());
  return 0;
}

}  // extern "C"
