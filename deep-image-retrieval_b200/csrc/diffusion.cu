// Diffusion re-ranking (manifold ranking, Zhou et al. NIPS 2003; Iscen et al. CVPR 2017): the mutual-kNN affinity
// graph of the database, a batched fp64 conjugate-gradient solve of (I - alpha S) f = y, and rank counting and exact
// top-k over the dense per-query f (dirb200_diffusion_*).  DESIGN.md section 4.7.
//
// Graph (dirb200_diffusion_graph), from the exact top-(k+1) lists of the database against itself:
//   nbr_sort_kernel      nn(i) = the first k list entries other than i (dropped by index, not position), sorted by
//                        index, with w_ij = max(s_ij, 0)^gamma
//   mutual_count_kernel  j in nn(i) is kept iff i in nn(j) (binary search in j's sorted list) -> per-row counts
//   scan_tile_kernel / scan_top_kernel / scan_out_kernel: row_ptr = inclusive scan of the counts (integers: exact)
//   fill_kernel          col ascending, val = w_ij, d_i = sum of the row in ascending j, u_i = 1 / sqrt(d_i) (0 if d_i = 0)
//   normalize_kernel     S_ij = A_ij * (u_i * u_j): the product order keeps S bit-exactly symmetric (s_ij == s_ji bit
//                        for bit, exact_dot_warp being symmetric in its operands)
// No atomics on values anywhere: a given input gives the same bits on every run.
//
// Solve (dirb200_diffusion_solve), Q queries stored [N][Q] row-major so that a nonzero gathers one contiguous Q-vector.
// Every reduction over rows runs over fixed blocks of RB rows: warp w of a block takes the rows w, w + 8, ... in order,
// the 8 warps are added in order, and the block partials are added by a fixed tree in cg_scalar_kernel.  Lane = query, so a
// query's arithmetic is the same whatever Q is and wherever it sits in the block: its f is bit-identical.
#include <limits.h>
#include <math.h>

#include <algorithm>

#include "block.cuh"
#include "common.h"

namespace dirb {
namespace {

constexpr int GRAPH_MAX_K = 2047;           // nbr_sort_kernel sorts a row of at most 2048 entries in shared memory
constexpr int SORT_CAP = 2048;
constexpr int SORT_THREADS = 128;

__global__ void __launch_bounds__(SORT_THREADS) nbr_sort_kernel(const int64_t* __restrict__ nn_idx,
                                                                const double* __restrict__ nn_score, int64_t N, int width,
                                                                int k, double gamma, int* __restrict__ nbr,
                                                                double* __restrict__ w, int* __restrict__ cnt) {
  __shared__ int ix[SORT_CAP];
  __shared__ double sw[SORT_CAP];
  __shared__ int s_n;
  const int64_t i = blockIdx.x;
  const int64_t* li = nn_idx + i * width;
  const double* ls = nn_score + i * width;
  const int lane = threadIdx.x & 31;
  if (threadIdx.x < 32) {                 // warp 0: keep the first k entries other than i and -1, in list order
    int base = 0;
    for (int e0 = 0; e0 < width && base < k; e0 += 32) {
      const int e = e0 + lane;
      const int64_t j = e < width ? li[e] : -1;
      const bool keep = j >= 0 && j != i;
      const unsigned m = __ballot_sync(0xffffffffu, keep);
      const int pos = base + __popc(m & ((1u << lane) - 1u));
      if (keep && pos < k) {
        ix[pos] = static_cast<int>(j);
        sw[pos] = pow(fmax(ls[e], 0.0), gamma);
      }
      base += __popc(m);
    }
    if (lane == 0) s_n = min(base, k);
  }
  __syncthreads();
  const int n = s_n;
  int P = 1;
  while (P < n) P <<= 1;
  for (int e = n + threadIdx.x; e < P; e += SORT_THREADS) ix[e] = INT_MAX;
  __syncthreads();
  block_bitonic_sort<SORT_THREADS>(ix, sw, P, [](int a, double, int b, double) { return a < b; });
  for (int e = threadIdx.x; e < k; e += SORT_THREADS) {
    nbr[i * k + e] = e < n ? ix[e] : -1;
    w[i * k + e] = e < n ? sw[e] : 0.0;
  }
  if (threadIdx.x == 0) cnt[i] = n;
}

__device__ __forceinline__ bool sorted_contains(const int* __restrict__ a, int n, int v) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (a[mid] < v) lo = mid + 1; else hi = mid;
  }
  return lo < n && a[lo] == v;
}

// one warp per row: mutual[i][e] = (nbr[i][e] lists i), mcnt[i] = how many do
__global__ void mutual_count_kernel(const int* __restrict__ nbr, const int* __restrict__ cnt, int64_t N, int k,
                                    uint8_t* __restrict__ mutual, int64_t* __restrict__ mcnt) {
  const int64_t i = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (i >= N) return;
  const int n = cnt[i];
  int c = 0;
  for (int e = lane; e < n; e += 32) {
    const int j = nbr[i * k + e];
    const bool m = sorted_contains(nbr + static_cast<int64_t>(j) * k, cnt[j], static_cast<int>(i));
    mutual[i * k + e] = m;
    c += m;
  }
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if (lane == 0) mcnt[i] = c;
}

// one warp per row: the mutual entries in ascending j -> col / val (= A_ij), then d_i in ascending j -> u_i
__global__ void fill_kernel(const int* __restrict__ nbr, const double* __restrict__ w, const int* __restrict__ cnt,
                            const uint8_t* __restrict__ mutual, int64_t N, int k, const int64_t* __restrict__ row_ptr,
                            int* __restrict__ col, double* __restrict__ val, double* __restrict__ u) {
  const int64_t i = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (i >= N) return;
  const int n = cnt[i];
  const int64_t r0 = row_ptr[i];
  int base = 0;
  for (int e0 = 0; e0 < n; e0 += 32) {
    const int e = e0 + lane;
    const bool m = e < n && mutual[i * k + e];
    const unsigned b = __ballot_sync(0xffffffffu, m);
    if (m) {
      const int64_t pos = r0 + base + __popc(b & ((1u << lane) - 1u));
      col[pos] = nbr[i * k + e];
      val[pos] = w[i * k + e];
    }
    base += __popc(b);
  }
  __syncwarp();
  if (lane == 0) {
    double d = 0.0;
    for (int64_t p = r0; p < r0 + base; ++p) d += val[p];
    u[i] = d > 0.0 ? 1.0 / sqrt(d) : 0.0;
  }
}

__global__ void normalize_kernel(const int64_t* __restrict__ row_ptr, const int* __restrict__ col, int64_t N,
                                 const double* __restrict__ u, double* __restrict__ val) {
  const int64_t i = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (i >= N) return;
  const double ui = u[i];
  for (int64_t p = row_ptr[i] + lane; p < row_ptr[i + 1]; p += 32) val[p] = val[p] * (ui * u[col[p]]);
}

// ------------------------------------------------------------------------------------------------ seeds
__global__ void seeds_kernel(const int64_t* __restrict__ idx, const double* __restrict__ score, int Q, int kq,
                             double gamma, int64_t N, double* __restrict__ y) {
  const int64_t t = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (t >= static_cast<int64_t>(Q) * kq) return;
  const int q = static_cast<int>(t / kq);
  const int64_t j = idx[t];
  if (j >= 0 && j < N) y[j * Q + q] = pow(fmax(score[t], 0.0), gamma);
}

// ------------------------------------------------------------------------------------------------ batched CG
constexpr int RB = 64;                      // rows per reduction block
constexpr int CG_WARPS = 8;
constexpr int CG_THREADS = 32 * CG_WARPS;
constexpr int RED_THREADS = 256;

// per-query scalars of the solve, in the workspace
struct CgState {
  double* yy;      // ||y||^2
  double* rr;      // ||r||^2 of the recurrence
  double* al;      // alpha_q of this iteration
  double* be;      // beta_q
  int* act;        // 1 while the query iterates
};

// acc of (warp, lane) over its rows -> part[b][q]: warps added in order
__device__ __forceinline__ void block_partial(double acc, double (*sh)[33], int warp, int lane, int q, int Q,
                                             double* __restrict__ part) {
  sh[warp][lane] = acc;
  __syncthreads();
  if (warp == 0 && q < Q) {
    double s = sh[0][lane];
#pragma unroll
    for (int w = 1; w < CG_WARPS; ++w) s += sh[w][lane];
    part[static_cast<int64_t>(blockIdx.x) * Q + q] = s;
  }
  __syncthreads();
}

// r = p = y, f = 0; part = ||y||^2 partials
__global__ void __launch_bounds__(CG_THREADS) cg_init_kernel(const double* __restrict__ y, int64_t N, int Q,
                                                             double* __restrict__ f, double* __restrict__ r,
                                                             double* __restrict__ p, double* __restrict__ part) {
  __shared__ double sh[CG_WARPS][33];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int q0 = 0; q0 < Q; q0 += 32) {
    const int q = q0 + lane;
    double acc = 0.0;
    for (int m = warp; m < RB; m += CG_WARPS) {
      const int64_t i = static_cast<int64_t>(blockIdx.x) * RB + m;
      if (i < N && q < Q) {
        const double v = y[i * Q + q];
        f[i * Q + q] = 0.0;
        r[i * Q + q] = v;
        p[i * Q + q] = v;
        acc += v * v;
      }
    }
    block_partial(acc, sh, warp, lane, q, Q, part);
  }
}

// ap = p - a S p (the nonzeros of a row in ascending column order); part = p . ap partials
__global__ void __launch_bounds__(CG_THREADS) cg_spmm_kernel(const int64_t* __restrict__ row_ptr,
                                                             const int* __restrict__ col, const double* __restrict__ val,
                                                             int64_t N, int Q, double a, const int* __restrict__ act,
                                                             const double* __restrict__ p, double* __restrict__ ap,
                                                             double* __restrict__ part) {
  __shared__ double sh[CG_WARPS][33];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int q0 = 0; q0 < Q; q0 += 32) {
    const int q = q0 + lane;
    const bool on = q < Q && act[q];
    double acc = 0.0;
    for (int m = warp; m < RB; m += CG_WARPS) {
      const int64_t i = static_cast<int64_t>(blockIdx.x) * RB + m;
      if (i >= N) break;
      double sp = 0.0;
      const int64_t e1 = row_ptr[i + 1];
      for (int64_t e = row_ptr[i]; e < e1; ++e) {
        const double v = val[e];
        const int64_t j = col[e];
        if (on) sp += v * p[j * Q + q];
      }
      if (on) {
        const double pi = p[i * Q + q];
        const double api = pi - a * sp;
        ap[i * Q + q] = api;
        acc += pi * api;
      }
    }
    block_partial(acc, sh, warp, lane, q, Q, part);
  }
}

// f += alpha p, r -= alpha ap; part = ||r||^2 partials
__global__ void __launch_bounds__(CG_THREADS) cg_update_kernel(int64_t N, int Q, CgState s, const double* __restrict__ p,
                                                               const double* __restrict__ ap, double* __restrict__ f,
                                                               double* __restrict__ r, double* __restrict__ part) {
  __shared__ double sh[CG_WARPS][33];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int q0 = 0; q0 < Q; q0 += 32) {
    const int q = q0 + lane;
    const bool on = q < Q && s.act[q];
    const double al = on ? s.al[q] : 0.0;
    double acc = 0.0;
    for (int m = warp; m < RB; m += CG_WARPS) {
      const int64_t i = static_cast<int64_t>(blockIdx.x) * RB + m;
      if (i < N && on) {
        const int64_t o = i * Q + q;
        f[o] = f[o] + al * p[o];
        const double rv = r[o] - al * ap[o];
        r[o] = rv;
        acc += rv * rv;
      }
    }
    block_partial(acc, sh, warp, lane, q, Q, part);
  }
}

// p = r + beta p
__global__ void __launch_bounds__(CG_THREADS) cg_pupdate_kernel(int64_t N, int Q, CgState s, const double* __restrict__ r,
                                                                double* __restrict__ p) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int q0 = 0; q0 < Q; q0 += 32) {
    const int q = q0 + lane;
    if (q >= Q || !s.act[q]) continue;
    const double be = s.be[q];
    for (int m = warp; m < RB; m += CG_WARPS) {
      const int64_t i = static_cast<int64_t>(blockIdx.x) * RB + m;
      if (i < N) p[i * Q + q] = r[i * Q + q] + be * p[i * Q + q];
    }
  }
}

// one block per query: the nb block partials added by a fixed tree (thread t takes the blocks t, t + 256, ... in order),
// then the step's scalars.  mode 0: ||y||^2 (start); 1: p.Ap -> alpha; 2: ||r||^2 -> beta, iteration count, stop test.
__global__ void __launch_bounds__(RED_THREADS) cg_scalar_kernel(const double* __restrict__ part, int nb, int Q, int mode,
                                                                double tol, CgState s, int* __restrict__ iters_out,
                                                                double* __restrict__ resid_out) {
  __shared__ double sh[RED_THREADS];
  const int q = blockIdx.x;
  if (mode != 0 && !s.act[q]) return;     // uniform over the block
  double v = 0.0;
  for (int b = threadIdx.x; b < nb; b += RED_THREADS) v += part[static_cast<int64_t>(b) * Q + q];
  sh[threadIdx.x] = v;
  __syncthreads();
  for (int h = RED_THREADS / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h) sh[threadIdx.x] += sh[threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x != 0) return;
  const double t = sh[0];
  if (mode == 0) {
    s.yy[q] = t;
    s.rr[q] = t;
    iters_out[q] = 0;
    resid_out[q] = sqrt(t);
    s.act[q] = t > 0.0 && !(sqrt(t) <= tol * sqrt(t));
  } else if (mode == 1) {
    s.al[q] = s.rr[q] / t;
  } else {
    s.be[q] = t / s.rr[q];
    s.rr[q] = t;
    iters_out[q] += 1;
    resid_out[q] = sqrt(t);
    if (sqrt(t) <= tol * sqrt(s.yy[q])) s.act[q] = 0;
  }
}

// ------------------------------------------------------------------------------------------------ rank counting
// Order of rule 6: f descending, ties -> lower index, -0 == +0: ranks_before on the keys fkey(f).

// one block per query: t_score of every target; the flagged targets sorted by rule 6 -> skey / srow / spos, nflag[q]
__global__ void rc_sort_kernel(const double* __restrict__ f, int64_t N, int Q, const int* __restrict__ t_off,
                               const int64_t* __restrict__ t_rows, const uint8_t* __restrict__ t_flags,
                               double* __restrict__ t_score, uint64_t* __restrict__ skey, int64_t* __restrict__ srow,
                               int* __restrict__ spos, int* __restrict__ nflag) {
  const int q = blockIdx.x;
  const int t0 = t_off[q], t1 = t_off[q + 1];
  int nf = 0;
  for (int a = t0 + threadIdx.x; a < t1; a += blockDim.x) {
    const int64_t ra = t_rows[a];
    const double fa = f[ra * Q + q];
    t_score[a] = fa;
    if (!t_flags[a]) continue;
    const uint64_t ka = fkey(fa);
    int pos = 0;
    for (int b = t0; b < t1; ++b) {
      if (b == a || !t_flags[b]) continue;
      const int64_t rb = t_rows[b];
      const uint64_t kb = fkey(f[rb * Q + q]);
      pos += ranks_before(kb, rb, ka, ra) || (kb == ka && rb == ra && b < a);
    }
    skey[t0 + pos] = ka;
    srow[t0 + pos] = ra;
    spos[t0 + pos] = a;
  }
  for (int a = t0 + threadIdx.x; a < t1; a += blockDim.x) nf += t_flags[a] != 0;
  for (int o = 16; o > 0; o >>= 1) nf += __shfl_xor_sync(0xffffffffu, nf, o);
  __shared__ int s_nf;
  if (threadIdx.x == 0) s_nf = 0;
  __syncthreads();
  if ((threadIdx.x & 31) == 0) atomicAdd(&s_nf, nf);
  __syncthreads();
  if (threadIdx.x == 0) nflag[q] = s_nf;
}

// grid (row chunks, Q): c(j) = the number of flagged targets not after row j (binary search); hist[q][c(j)] += 1.
// Row j ranks before exactly the targets at sorted positions >= c(j).
constexpr int RC_ROWS = 8192;
constexpr int RC_THREADS = 256;
__global__ void __launch_bounds__(RC_THREADS) rc_count_kernel(const double* __restrict__ f, int64_t N, int Q,
                                                              const int* __restrict__ t_off,
                                                              const uint64_t* __restrict__ skey,
                                                              const int64_t* __restrict__ srow,
                                                              const int* __restrict__ nflag,
                                                              unsigned long long* __restrict__ hist) {
  extern __shared__ unsigned int h[];
  const int q = blockIdx.y;
  const int nf = nflag[q];
  if (nf == 0) return;                    // uniform
  const int t0 = t_off[q];
  for (int c = threadIdx.x; c <= nf; c += RC_THREADS) h[c] = 0u;
  __syncthreads();
  const int64_t j0 = static_cast<int64_t>(blockIdx.x) * RC_ROWS;
  const int64_t j1 = min(N, j0 + RC_ROWS);
  for (int64_t j = j0 + threadIdx.x; j < j1; j += RC_THREADS) {
    const uint64_t kj = fkey(f[j * Q + q]);
    int lo = 0, hi = nf;                  // first sorted target that row j ranks before
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (ranks_before(kj, j, skey[t0 + mid], srow[t0 + mid])) hi = mid; else lo = mid + 1;
    }
    atomicAdd(&h[lo], 1u);
  }
  __syncthreads();
  for (int c = threadIdx.x; c < nf; c += RC_THREADS)
    if (h[c]) atomicAdd(hist + t0 + q + c, static_cast<unsigned long long>(h[c]));
}

// one thread per query: above[target at sorted position s] = sum_{c <= s} hist[c]
__global__ void rc_prefix_kernel(int Q, const int* __restrict__ t_off, const int* __restrict__ spos,
                                 const int* __restrict__ nflag, const unsigned long long* __restrict__ hist,
                                 int64_t* __restrict__ above) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= Q) return;
  const int t0 = t_off[q];
  unsigned long long acc = 0;
  for (int s = 0; s < nflag[q]; ++s) {
    acc += hist[t0 + q + s];
    above[spos[t0 + s]] = static_cast<int64_t>(acc);
  }
}

// row_ptr[i + 1] = sum_{i' <= i} mcnt[i'] in tiles of SCAN_TILE rows: tile totals, their exclusive scan, then each
// tile's own scan plus its offset
constexpr int SCAN_THREADS = 256, SCAN_PER = 8, SCAN_TILE = SCAN_THREADS * SCAN_PER;

// v = the thread's running sums of its SCAN_PER counts; returns the sum over the tile's earlier threads
__device__ __forceinline__ int64_t tile_scan(const int64_t* __restrict__ c, int64_t N, int64_t (&v)[SCAN_PER],
                                             int64_t* warp_sums, int64_t& total) {
  const int64_t i0 = static_cast<int64_t>(blockIdx.x) * SCAN_TILE + threadIdx.x * SCAN_PER;
  int64_t s = 0;
#pragma unroll
  for (int e = 0; e < SCAN_PER; ++e) {
    s += i0 + e < N ? c[i0 + e] : 0;
    v[e] = s;
  }
  return block_scan(s, warp_sums, &total) - s;
}

__global__ void __launch_bounds__(SCAN_THREADS) scan_tile_kernel(const int64_t* __restrict__ c, int64_t N,
                                                                 int64_t* __restrict__ tile_sum) {
  __shared__ int64_t warp_sums[SCAN_THREADS / 32];
  int64_t v[SCAN_PER], total;
  tile_scan(c, N, v, warp_sums, total);
  if (threadIdx.x == 0) tile_sum[blockIdx.x] = total;
}

__global__ void scan_top_kernel(int64_t* __restrict__ tile_sum, int nt) {
  int64_t acc = 0;
  for (int t = 0; t < nt; ++t) {
    const int64_t v = tile_sum[t];
    tile_sum[t] = acc;
    acc += v;
  }
}

__global__ void __launch_bounds__(SCAN_THREADS) scan_out_kernel(const int64_t* __restrict__ c, int64_t N,
                                                                const int64_t* __restrict__ tile_off,
                                                                int64_t* __restrict__ row_ptr) {
  __shared__ int64_t warp_sums[SCAN_THREADS / 32];
  int64_t v[SCAN_PER], total;
  const int64_t excl = tile_scan(c, N, v, warp_sums, total) + tile_off[blockIdx.x];
  const int64_t i0 = static_cast<int64_t>(blockIdx.x) * SCAN_TILE + threadIdx.x * SCAN_PER;
#pragma unroll
  for (int e = 0; e < SCAN_PER; ++e)
    if (i0 + e < N) row_ptr[i0 + e + 1] = excl + v[e];
}

// graph workspace: nbr int32 [N][k], w fp64 [N][k], cnt int32 [N], mutual uint8 [N][k], mcnt int64 [N], u fp64 [N],
// scan tile sums
struct GraphWs {
  int* nbr; double* w; int* cnt; uint8_t* mutual; int64_t* mcnt; double* u; int64_t* tiles; size_t total;
};
GraphWs graph_ws(void* base, int64_t N, int k) {
  Carver c(base);
  GraphWs g;
  g.nbr = c.take<int>(size_t(N) * k);
  g.w = c.take<double>(size_t(N) * k);
  g.cnt = c.take<int>(N);
  g.mutual = c.take<uint8_t>(size_t(N) * k);
  g.mcnt = c.take<int64_t>(N);
  g.u = c.take<double>(N);
  g.tiles = c.take<int64_t>(ceil_div(N, SCAN_TILE));
  g.total = c.used;
  return g;
}

int64_t cg_blocks(int64_t N) { return ceil_div(N, RB); }

struct SolveWs { double *r, *p, *ap, *part; CgState s; size_t total; };
SolveWs solve_ws(void* base, int64_t N, int Q) {
  Carver c(base);
  SolveWs w;
  const size_t nq = size_t(N) * Q;
  w.r = c.take<double>(nq);
  w.p = c.take<double>(nq);
  w.ap = c.take<double>(nq);
  w.part = c.take<double>(size_t(cg_blocks(N)) * Q);
  w.s.yy = c.take<double>(Q);
  w.s.rr = c.take<double>(Q);
  w.s.al = c.take<double>(Q);
  w.s.be = c.take<double>(Q);
  w.s.act = c.take<int>(Q);
  w.total = c.used;
  return w;
}

struct RankWs { uint64_t* skey; int64_t* srow; int* spos; int* nflag; unsigned long long* hist; size_t hist_bytes, total; };
RankWs rank_ws(void* base, int Q, int T) {
  Carver c(base);
  RankWs w;
  w.skey = c.take<uint64_t>(T);
  w.srow = c.take<int64_t>(T);
  w.spos = c.take<int>(T);
  w.nflag = c.take<int>(Q);
  w.hist_bytes = (size_t(T) + Q) * 8;
  w.hist = c.take<unsigned long long>(size_t(T) + Q);
  w.total = c.used;
  return w;
}

// ------------------------------------------------------------------------------------------------ dense-row top-k
// Exact top-k of each column of f under rule 6.  A radix select, 8 bits per pass, finds the k-th key K and how many of
// the k go to rows with key == K (passes 0-7 over the key); passes 8-11 select, among the rows with key == K, the
// lowest indices needed (digits of ~index).  tk_compact_kernel then gathers exactly k (row, f) pairs per query, which
// sort_runs_merge (the deep search's run sort and rank merge, search.cu) orders by (f desc, row asc); -0 == +0 there
// as in the key, since the merge compares doubles.
constexpr int TK_ROWS = 8192;
constexpr int TK_THREADS = 256;

__global__ void __launch_bounds__(TK_THREADS) tk_hist_kernel(const double* __restrict__ f, int64_t N, int Q, int pass,
                                                             const uint64_t* __restrict__ kp,
                                                             const uint32_t* __restrict__ vp,
                                                             unsigned long long* __restrict__ hist) {
  __shared__ unsigned int h[256];
  const int q = blockIdx.y;
  h[threadIdx.x] = 0u;
  __syncthreads();
  const uint64_t pk = kp[q];
  const uint32_t pv = vp[q];
  const int64_t j0 = static_cast<int64_t>(blockIdx.x) * TK_ROWS;
  const int64_t j1 = min(N, j0 + TK_ROWS);
  for (int64_t j = j0 + threadIdx.x; j < j1; j += TK_THREADS) {
    const uint64_t key = fkey(f[j * Q + q]);
    if (pass < 8) {
      const int shift = 56 - 8 * pass;
      if (pass == 0 || (key >> (shift + 8)) == (pk >> (shift + 8))) atomicAdd(&h[(key >> shift) & 255u], 1u);
    } else if (key == pk) {
      const uint32_t v = ~static_cast<uint32_t>(j);
      const int shift = 24 - 8 * (pass - 8);
      if (pass == 8 || (v >> (shift + 8)) == (pv >> (shift + 8))) atomicAdd(&h[(v >> shift) & 255u], 1u);
    }
  }
  __syncthreads();
  if (h[threadIdx.x]) atomicAdd(hist + static_cast<int64_t>(q) * 256 + threadIdx.x, static_cast<unsigned long long>(h[threadIdx.x]));
}

// one thread per query: the digit holding the r-th largest candidate; r becomes its rank among that digit's rows
__global__ void tk_pick_kernel(int Q, int pass, unsigned long long* __restrict__ hist, uint64_t* __restrict__ kp,
                               uint32_t* __restrict__ vp, long long* __restrict__ r) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= Q) return;
  unsigned long long* h = hist + static_cast<int64_t>(q) * 256;
  long long rr = r[q];
  int b = 255;
  for (; b > 0; --b) {
    const long long c = static_cast<long long>(h[b]);
    if (rr <= c) break;
    rr -= c;
  }
  if (pass < 8) kp[q] |= static_cast<uint64_t>(b) << (56 - 8 * pass);
  else vp[q] |= static_cast<uint32_t>(b) << (24 - 8 * (pass - 8));
  r[q] = rr;
  for (int i = 0; i < 256; ++i) h[i] = 0ull;
}

// rows with key > K, or key == K and index <= ~v: exactly k per query -> (rows, sc)[q * cap2 + pos]
__global__ void __launch_bounds__(TK_THREADS) tk_compact_kernel(const double* __restrict__ f, int64_t N, int Q,
                                                                const uint64_t* __restrict__ kp,
                                                                const uint32_t* __restrict__ vp, int cap2,
                                                                int* __restrict__ cnt, int* __restrict__ rows,
                                                                double* __restrict__ sc) {
  const int q = blockIdx.y;
  const uint64_t K = kp[q];
  const uint32_t last = ~vp[q];
  const int64_t j0 = static_cast<int64_t>(blockIdx.x) * TK_ROWS;
  const int64_t j1 = min(N, j0 + TK_ROWS);
  for (int64_t j = j0 + threadIdx.x; j < j1; j += TK_THREADS) {
    const double v = f[j * Q + q];
    const uint64_t key = fkey(v);
    if (key > K || (key == K && static_cast<uint32_t>(j) <= last)) {
      const int pos = atomicAdd(cnt + q, 1);
      if (pos < cap2) {
        rows[static_cast<int64_t>(q) * cap2 + pos] = static_cast<int>(j);
        sc[static_cast<int64_t>(q) * cap2 + pos] = v;
      }
    }
  }
}

struct TopkWs {
  unsigned long long* hist; uint64_t* kp; uint32_t* vp; long long* r; int* cnt; SortScratch s;
  unsigned long long* status; size_t total;
};
TopkWs topk_ws(void* base, int Q, int cap2) {
  Carver c(base);
  TopkWs w;
  w.hist = c.take<unsigned long long>(size_t(Q) * 256);
  w.kp = c.take<uint64_t>(Q);
  w.vp = c.take<uint32_t>(Q);
  w.r = c.take<long long>(Q);
  w.cnt = c.take<int>(Q);
  w.s = take_sort_scratch(c, Q, cap2);
  w.status = c.take<unsigned long long>(8);
  w.total = c.used;
  return w;
}

__global__ void tk_init_kernel(int Q, int k, uint64_t* __restrict__ kp, uint32_t* __restrict__ vp, long long* __restrict__ r,
                               int* __restrict__ cnt) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= Q) return;
  kp[q] = 0;
  vp[q] = 0;
  r[q] = k;
  cnt[q] = 0;
}

constexpr int RC_MAX_FLAGGED = 12000;       // the per-block histogram (nf + 1 counters) stays within 48 KB

// the graph launches of dirb200_diffusion_graph; a_dev / u_dev (both or neither) also receive A (val before
// normalize_kernel, N * k capacity) and u
int diffusion_graph(const int64_t* nn_idx_dev, const double* nn_score_dev, int64_t N, int width, int k, double gamma,
                    void* ws_dev, int64_t* row_ptr_dev, int* col_dev, double* val_dev, double* a_dev, double* u_dev,
                    void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DIRB_REQUIRE(N >= 1 && N < INT_MAX && k >= 1 && width >= 1 && width <= k + 1, DIRB200_EINVAL,
               "diffusion_graph: bad sizes N %lld, width %d, k %d", (long long)N, width, k);
  DIRB_REQUIRE(k <= GRAPH_MAX_K, DIRB200_ENOTSUP, "diffusion_graph: k %d exceeds %d", k, GRAPH_MAX_K);
  DIRB_REQUIRE(gamma > 0.0, DIRB200_EINVAL, "diffusion_graph: gamma must be > 0 (got %g)", gamma);
  DIRB_REQUIRE(nn_idx_dev && nn_score_dev && ws_dev && row_ptr_dev && col_dev && val_dev, DIRB200_EINVAL,
               "diffusion_graph: null argument");
  DIRB_TRY(require_sm90());
  GraphWs g = graph_ws(ws_dev, N, k);
  const unsigned wblocks = static_cast<unsigned>(ceil_div(N * 32, 256));
  nbr_sort_kernel<<<static_cast<unsigned>(N), SORT_THREADS, 0, stream>>>(nn_idx_dev, nn_score_dev, N, width, k, gamma,
                                                                          g.nbr, g.w, g.cnt);
  mutual_count_kernel<<<wblocks, 256, 0, stream>>>(g.nbr, g.cnt, N, k, g.mutual, g.mcnt);
  DIRB_CUDA(cudaMemsetAsync(row_ptr_dev, 0, 8, stream));
  const int nt = static_cast<int>(ceil_div(N, SCAN_TILE));
  scan_tile_kernel<<<nt, SCAN_THREADS, 0, stream>>>(g.mcnt, N, g.tiles);
  scan_top_kernel<<<1, 1, 0, stream>>>(g.tiles, nt);
  scan_out_kernel<<<nt, SCAN_THREADS, 0, stream>>>(g.mcnt, N, g.tiles, row_ptr_dev);
  fill_kernel<<<wblocks, 256, 0, stream>>>(g.nbr, g.w, g.cnt, g.mutual, N, k, row_ptr_dev, col_dev, val_dev, g.u);
  if (a_dev) {
    DIRB_CUDA(cudaMemcpyAsync(a_dev, val_dev, size_t(N) * k * 8, cudaMemcpyDeviceToDevice, stream));
    DIRB_CUDA(cudaMemcpyAsync(u_dev, g.u, size_t(N) * 8, cudaMemcpyDeviceToDevice, stream));
  }
  normalize_kernel<<<wblocks, 256, 0, stream>>>(row_ptr_dev, col_dev, N, g.u, val_dev);
  count_launch(7);
  DIRB_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace
}  // namespace dirb

using namespace dirb;

extern "C" {

size_t dirb200_diffusion_graph_workspace_bytes(int64_t N, int k) {
  if (N < 1 || k < 1) return 0;
  return graph_ws(nullptr, N, k).total;
}

int dirb200_diffusion_graph(const int64_t* nn_idx_dev, const double* nn_score_dev, int64_t N, int width, int k,
                            double gamma, void* ws_dev, int64_t* row_ptr_dev, int* col_dev, double* val_dev,
                            void* stream) {
  return diffusion_graph(nn_idx_dev, nn_score_dev, N, width, k, gamma, ws_dev, row_ptr_dev, col_dev, val_dev, nullptr,
                         nullptr, stream);
}

int dirb200_diffusion_graph_weights(const int64_t* nn_idx_dev, const double* nn_score_dev, int64_t N, int width, int k,
                                    double gamma, void* ws_dev, int64_t* row_ptr_dev, int* col_dev, double* val_dev,
                                    double* a_dev, double* u_dev, void* stream) {
  DIRB_REQUIRE(a_dev && u_dev, DIRB200_EINVAL, "diffusion_graph_weights: null argument");
  return diffusion_graph(nn_idx_dev, nn_score_dev, N, width, k, gamma, ws_dev, row_ptr_dev, col_dev, val_dev, a_dev,
                         u_dev, stream);
}

int dirb200_diffusion_seeds(const int64_t* idx_dev, const double* score_dev, int Q, int kq, double gamma, int64_t N,
                            double* y_dev, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DIRB_REQUIRE(Q >= 1 && kq >= 1 && N >= 1, DIRB200_EINVAL, "diffusion_seeds: bad sizes Q %d, kq %d, N %lld", Q, kq,
               (long long)N);
  DIRB_REQUIRE(gamma > 0.0, DIRB200_EINVAL, "diffusion_seeds: gamma must be > 0 (got %g)", gamma);
  DIRB_REQUIRE(idx_dev && score_dev && y_dev, DIRB200_EINVAL, "diffusion_seeds: null argument");
  DIRB_TRY(require_sm90());
  DIRB_CUDA(cudaMemsetAsync(y_dev, 0, size_t(N) * Q * 8, stream));
  const int64_t n = static_cast<int64_t>(Q) * kq;
  seeds_kernel<<<static_cast<unsigned>(ceil_div(n, 256)), 256, 0, stream>>>(idx_dev, score_dev, Q, kq, gamma, N, y_dev);
  count_launch();
  DIRB_CUDA(cudaGetLastError());
  return 0;
}

size_t dirb200_diffusion_solve_workspace_bytes(int64_t N, int Q) {
  if (N < 1 || Q < 1) return 0;
  return solve_ws(nullptr, N, Q).total;
}

int dirb200_diffusion_solve(const int64_t* row_ptr_dev, const int* col_dev, const double* val_dev, int64_t N,
                            const double* y_dev, int Q, double alpha, int iters, double tol, void* ws_dev, double* f_dev,
                            int* iters_dev, double* resid_dev, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DIRB_REQUIRE(N >= 1 && Q >= 1, DIRB200_EINVAL, "diffusion_solve: bad sizes N %lld, Q %d", (long long)N, Q);
  DIRB_REQUIRE(alpha >= 0.0 && alpha < 1.0 && iters >= 1 && tol >= 0.0, DIRB200_EINVAL,
               "diffusion_solve: need 0 <= alpha < 1, iters >= 1, tol >= 0 (got %g, %d, %g)", alpha, iters, tol);
  DIRB_REQUIRE(row_ptr_dev && col_dev && val_dev && y_dev && ws_dev && f_dev && iters_dev && resid_dev, DIRB200_EINVAL,
               "diffusion_solve: null argument");
  DIRB_TRY(require_sm90());
  SolveWs w = solve_ws(ws_dev, N, Q);
  const int nb = static_cast<int>(cg_blocks(N));
  const unsigned g = static_cast<unsigned>(nb);
  cg_init_kernel<<<g, CG_THREADS, 0, stream>>>(y_dev, N, Q, f_dev, w.r, w.p, w.part);
  cg_scalar_kernel<<<Q, RED_THREADS, 0, stream>>>(w.part, nb, Q, 0, tol, w.s, iters_dev, resid_dev);
  for (int it = 0; it < iters; ++it) {
    cg_spmm_kernel<<<g, CG_THREADS, 0, stream>>>(row_ptr_dev, col_dev, val_dev, N, Q, alpha, w.s.act, w.p, w.ap, w.part);
    cg_scalar_kernel<<<Q, RED_THREADS, 0, stream>>>(w.part, nb, Q, 1, tol, w.s, iters_dev, resid_dev);
    cg_update_kernel<<<g, CG_THREADS, 0, stream>>>(N, Q, w.s, w.p, w.ap, f_dev, w.r, w.part);
    cg_scalar_kernel<<<Q, RED_THREADS, 0, stream>>>(w.part, nb, Q, 2, tol, w.s, iters_dev, resid_dev);
    if (it + 1 < iters) cg_pupdate_kernel<<<g, CG_THREADS, 0, stream>>>(N, Q, w.s, w.r, w.p);
  }
  count_launch(2 + 5 * iters - 1);
  DIRB_CUDA(cudaGetLastError());
  return 0;
}

size_t dirb200_diffusion_rank_count_workspace_bytes(int Q, int T) {
  if (Q < 1 || T < 0) return 0;
  return rank_ws(nullptr, Q, T).total;
}

int dirb200_diffusion_rank_count(const double* f_dev, int64_t N, int Q, const int* t_off_host, const int* t_off_dev,
                                 const int64_t* t_rows_dev, const uint8_t* t_flags_dev, int T, void* ws_dev,
                                 double* t_score_dev, int64_t* above_dev, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DIRB_REQUIRE(N >= 1 && Q >= 1 && T >= 0, DIRB200_EINVAL, "diffusion_rank_count: bad sizes N %lld, Q %d, T %d",
               (long long)N, Q, T);
  DIRB_REQUIRE(f_dev && t_off_host && t_off_dev && ws_dev && (T == 0 || (t_rows_dev && t_flags_dev && t_score_dev && above_dev)),
               DIRB200_EINVAL, "diffusion_rank_count: null argument");
  DIRB_REQUIRE(t_off_host[0] == 0 && t_off_host[Q] == T, DIRB200_EINVAL, "diffusion_rank_count: t_off must run from 0 to T");
  int max_t = 0;
  for (int q = 0; q < Q; ++q) {
    DIRB_REQUIRE(t_off_host[q + 1] >= t_off_host[q], DIRB200_EINVAL, "diffusion_rank_count: t_off must not decrease");
    max_t = std::max(max_t, t_off_host[q + 1] - t_off_host[q]);
  }
  DIRB_REQUIRE(Q <= 65535, DIRB200_ENOTSUP, "diffusion_rank_count: at most 65535 queries per call (got %d)", Q);
  DIRB_REQUIRE(max_t <= RC_MAX_FLAGGED, DIRB200_ENOTSUP, "diffusion_rank_count: %d targets for one query exceed %d", max_t,
               RC_MAX_FLAGGED);
  DIRB_TRY(require_sm90());
  if (T == 0) return 0;
  RankWs w = rank_ws(ws_dev, Q, T);
  DIRB_CUDA(cudaMemsetAsync(w.hist, 0, w.hist_bytes, stream));
  DIRB_CUDA(cudaMemsetAsync(above_dev, 0, size_t(T) * 8, stream));
  rc_sort_kernel<<<Q, 256, 0, stream>>>(f_dev, N, Q, t_off_dev, t_rows_dev, t_flags_dev, t_score_dev, w.skey, w.srow,
                                        w.spos, w.nflag);
  rc_count_kernel<<<dim3(static_cast<unsigned>(ceil_div(N, RC_ROWS)), Q), RC_THREADS, (max_t + 1) * 4, stream>>>(
      f_dev, N, Q, t_off_dev, w.skey, w.srow, w.nflag, w.hist);
  rc_prefix_kernel<<<static_cast<unsigned>(ceil_div(Q, 128)), 128, 0, stream>>>(Q, t_off_dev, w.spos, w.nflag, w.hist,
                                                                                 above_dev);
  count_launch(3);
  DIRB_CUDA(cudaGetLastError());
  return 0;
}


size_t dirb200_diffusion_topk_workspace_bytes(int Q, int k) {
  if (Q < 1 || k < 1) return 0;
  return topk_ws(nullptr, Q, sort_run_cap(k)).total;
}

int dirb200_diffusion_topk(const double* f_dev, int64_t N, int Q, int k, void* ws_dev, double* scores_dev,
                           int64_t* idx_dev, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DIRB_REQUIRE(N >= 1 && N < INT_MAX && Q >= 1 && k >= 1 && k <= N, DIRB200_EINVAL,
               "diffusion_topk: need N >= 1, Q >= 1, 1 <= k <= N (got N %lld, Q %d, k %d)", (long long)N, Q, k);
  DIRB_REQUIRE(Q <= 65535, DIRB200_ENOTSUP, "diffusion_topk: at most 65535 queries per call (got %d)", Q);
  DIRB_REQUIRE(f_dev && ws_dev && scores_dev && idx_dev, DIRB200_EINVAL, "diffusion_topk: null argument");
  DIRB_TRY(require_sm90());
  const int cap2 = sort_run_cap(k);
  TopkWs w = topk_ws(ws_dev, Q, cap2);
  DIRB_CUDA(cudaMemsetAsync(w.hist, 0, size_t(Q) * 256 * 8, stream));
  tk_init_kernel<<<static_cast<unsigned>(ceil_div(Q, 128)), 128, 0, stream>>>(Q, k, w.kp, w.vp, w.r, w.cnt);
  const dim3 grid(static_cast<unsigned>(ceil_div(N, TK_ROWS)), Q);
  for (int pass = 0; pass < 12; ++pass) {
    tk_hist_kernel<<<grid, TK_THREADS, 0, stream>>>(f_dev, N, Q, pass, w.kp, w.vp, w.hist);
    tk_pick_kernel<<<static_cast<unsigned>(ceil_div(Q, 128)), 128, 0, stream>>>(Q, pass, w.hist, w.kp, w.vp, w.r);
  }
  tk_compact_kernel<<<grid, TK_THREADS, 0, stream>>>(f_dev, N, Q, w.kp, w.vp, cap2, w.cnt, w.s.rows, w.s.sc);
  count_launch(26);
  DIRB_CUDA(cudaGetLastError());
  return sort_runs_merge(w.s.rows, w.cnt, cap2, w.s.sc, w.s.run_ix, Q, k, 0, w.status, scores_dev, idx_dev, stream);
}

}  // extern "C"
