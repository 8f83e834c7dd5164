// Column sums and the centred Gram matrix in fp64: the statistics of a PCA fit (dirb200_col_sums_f64, dirb200_gram_f64).
//
// sklearn's PCA.fit (_pca.py, _fit_full) either takes the SVD of the centred data on the host or, with
// svd_solver='covariance_eigh', forms X^T X - n m m^T and diagonalises it.  Here the covariance comes from the GPU:
//
//   1. column sums (col_sum_part_kernel, col_sum_reduce_kernel): the rows are cut into P blocks (P a function of N
//      only), one fp64 partial per block and column, added in block order.  Fixed order: bit-identical on every run.
//   2. Gram G[i][j] = sum_r (x[r][i] - m[i]) (x[r][j] - m[j]) (gram_tile_kernel, gram_reduce_kernel).  A GEMM A^T A
//      with the rows as the K dimension, on fp64 tensor cores (dmma.cuh): fp32 rows come to shared memory by cp.async
//      and are widened to fp64 in shared memory before the fragments are loaded; the centring x - m happens there, in
//      fp64 (one rounding per element, the same as numpy's float64(x) - mean).  The
//      uncentred form X^T X - n m m^T cancels catastrophically once |m| >> the spread of the data (descriptors have
//      means of the order of their spread); centred products lose nothing.
//      Only the 128 x 128 tiles on or above the diagonal are computed.  Split-K over the rows: S splits, S a function
//      of (N, D) only (never of the SM count), each writing its partial tile to scratch; the reduction adds the S
//      partials in split order and mirrors each tile into the lower triangle.  No atomics: a given input gives
//      bit-identical output on every run and every H100, and the matrix is exactly symmetric.
//      The partials live in the per-device scratch (ops.cu), bounded by GRAM_WS_BYTES: that bounds D (D_MAX).
//
// Both entry points ADD into the caller's buffers, so rows can be fed in chunks.
#include <math.h>

#include <algorithm>
#include <atomic>

#include "conv.h"
#include "dmma.cuh"

namespace dirb {
namespace {

// Gram tile: 128 x 128 outputs per CTA, 16 warps of 32 x 32 (4 x 4), K staged 32 rows at a time.  fp32 rows arrive
// by cp.async in GST stages ([row][feature], stride GLD); once a stage has landed, the CTA widens it to fp64, subtracts
// the means and zeroes the rows past the split's end, into one fp64 stage ([row][feature], stride GLD64 = 132 = 4 mod
// 16 doubles: the fragment loads, 8 features x 4 rows per warp, are two conflict-free wavefronts).  Each element is
// converted once per CTA instead of once per warp that reads it, and the fragments are plain 64-bit loads.
constexpr int GT = 128, GK = 32, GST = 3, GLD = GT + 8, GLD64 = GT + 4, G_THREADS = 512;
constexpr int G_SMEM = GST * 2 * GK * GLD * 4 + 2 * GK * GLD64 * 8;   // 104448 + 67584 bytes
constexpr size_t GRAM_TILE_BYTES = size_t(GT) * GT * 8;
constexpr size_t GRAM_WS_BYTES = size_t(256) << 20;                  // partial tiles of all splits
constexpr int GRAM_MAX_TILES = static_cast<int>(GRAM_WS_BYTES / GRAM_TILE_BYTES);   // 2048 upper tiles: T <= 63
constexpr int D_MAX = 63 * GT;                                       // 8064
static_assert((D_MAX / GT) * (D_MAX / GT + 1) / 2 <= GRAM_MAX_TILES, "one split of D_MAX must fit the workspace");
constexpr int64_t GRAM_SPLIT_ROWS = 1024;                            // a split takes at least this many rows
// Column sums: at most CS_MAX_PARTS row blocks of at least CS_ROWS rows.
constexpr int64_t CS_ROWS = 4096;
constexpr int CS_MAX_PARTS = 1024;

__device__ __forceinline__ void upper_tile(int t, int T, int& bi, int& bj) {
  bi = 0;
  while (t >= T - bi) {
    t -= T - bi;
    ++bi;
  }
  bj = bi + t;
}

// One stage of GK centred fp64 rows: acc += A^T B for this warp's 32 x 32 outputs.
__device__ __forceinline__ void gram_stage(double (&acc)[2][4][4], const double* __restrict__ a_s,
                                           const double* __restrict__ b_s, int g, int t4, int wm, int wn) {
#pragma unroll
  for (int kk = 0; kk < GK; kk += 16) {
    double a[2][8];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) {
      const double* p = a_s + (kk + t4) * GLD64 + wm * 32 + mt * 16 + g;
#pragma unroll
      for (int i = 0; i < 8; ++i) a[mt][i] = p[(i >> 1) * 4 * GLD64 + (i & 1) * 8];
    }
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
      double b[4];
      const double* p = b_s + (kk + t4) * GLD64 + wn * 32 + nt * 8 + g;
#pragma unroll
      for (int i = 0; i < 4; ++i) b[i] = p[4 * i * GLD64];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) dmma16816(acc[mt][nt], a[mt], b);
    }
  }
}

// grid (upper tiles, splits).  Partial tile of split s, tile t -> part[(s * tiles + t) * GT * GT], row-major 128 x 128.
__global__ void __launch_bounds__(G_THREADS, 1) gram_tile_kernel(const float* __restrict__ x, int64_t N, int D,
                                                                 const double* __restrict__ mean, int64_t rows_per_split,
                                                                 int T, double* __restrict__ part) {
  extern __shared__ __align__(16) float smem[];
  float* sA = smem;                                   // [GST][GK][GLD]  fp32, features i0 ..
  float* sB = smem + GST * GK * GLD;                  // [GST][GK][GLD]  fp32, features j0 ..
  double* sA64 = reinterpret_cast<double*>(smem + 2 * GST * GK * GLD);   // [GK][GLD64]  centred fp64
  double* sB64 = sA64 + GK * GLD64;
  int bi, bj;
  upper_tile(blockIdx.x, T, bi, bj);
  const int i0 = bi * GT, j0 = bj * GT;
  const int64_t r0 = static_cast<int64_t>(blockIdx.y) * rows_per_split;
  const int64_t r1 = min(N, r0 + rows_per_split);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = lane >> 2, t4 = lane & 3;
  const int wm = warp & 3, wn = warp >> 2;

  auto load_stage = [&](int s, int64_t k0) {
#pragma unroll
    for (int i = 0; i < (GK * GT / 4) / G_THREADS; ++i) {
      const int c = tid + i * G_THREADS, row = c >> 5, c4 = c & 31;
      const int64_t gr = k0 + row;
      const bool okr = gr < r1;
      const int fa = i0 + c4 * 4, fb = j0 + c4 * 4;   // D % 4 == 0: a float4 is wholly inside or outside
      cp_async16(sA + (s * GK + row) * GLD + c4 * 4, x + (okr && fa < D ? gr * D + fa : 0), okr && fa < D);
      cp_async16(sB + (s * GK + row) * GLD + c4 * 4, x + (okr && fb < D ? gr * D + fb : 0), okr && fb < D);
    }
  };

  // widening: thread -> one feature column (A for tid % 256 < 128, else B) and the rows tid / 256 + 2 q.  Features
  // past D hold 0 with a mean of 0, and rows past the split's end are written as 0: neither contributes.
  const int cv_col = tid & (2 * GT - 1), cv_row = tid >> 8;
  const bool cv_b = cv_col >= GT;
  const int cv_f = (cv_b ? j0 - GT : i0) + cv_col;
  const double cv_mean = cv_f < D ? mean[cv_f] : 0.0;
  const float* cv_src = (cv_b ? sB - GT : sA) + cv_col;
  double* cv_dst = (cv_b ? sB64 - GT : sA64) + cv_col;

  double acc[2][4][4];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int k = 0; k < 4; ++k) acc[i][j][k] = 0.0;

  const int nk = static_cast<int>((r1 - r0 + GK - 1) / GK);
#pragma unroll
  for (int s = 0; s < GST - 1; ++s) {
    if (s < nk) load_stage(s, r0 + static_cast<int64_t>(s) * GK);
    cp_async_commit();
  }
  for (int kt = 0; kt < nk; ++kt) {
    cp_async_wait<GST - 2>();
    __syncthreads();      // stage kt landed; stage kt-1 and the fp64 stage are no longer read by anyone
    if (kt + GST - 1 < nk) load_stage((kt + GST - 1) % GST, r0 + static_cast<int64_t>(kt + GST - 1) * GK);
    cp_async_commit();
    const int64_t valid = r1 - (r0 + static_cast<int64_t>(kt) * GK);
    const float* src = cv_src + (kt % GST) * GK * GLD;
#pragma unroll
    for (int q = 0; q < GK / 2; ++q) {
      const int row = cv_row + 2 * q;
      cv_dst[row * GLD64] = row < valid ? static_cast<double>(src[row * GLD]) - cv_mean : 0.0;
    }
    __syncthreads();      // the fp64 stage is complete
    gram_stage(acc, sA64, sB64, g, t4, wm, wn);
  }
  cp_async_wait<0>();

  double* out = part + (static_cast<int64_t>(blockIdx.y) * gridDim.x + blockIdx.x) * (GT * GT);
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int m = wm * 32 + mt * 16 + g + 8 * h, n = wn * 32 + nt * 8 + 2 * t4;
        *reinterpret_cast<double2*>(out + m * GT + n) = make_double2(acc[mt][nt][2 * h], acc[mt][nt][2 * h + 1]);
      }
}

// grid (upper tiles, GT * GT / 1024), 256 threads x 4 elements.  gram[i][j] += sum over splits in order, for i <= j,
// and the same value into gram[j][i] (on a diagonal tile only the elements with m <= n are read).
__global__ void __launch_bounds__(256) gram_reduce_kernel(const double* __restrict__ part, int S, int T, int D,
                                                          double* __restrict__ gram) {
  int bi, bj;
  upper_tile(blockIdx.x, T, bi, bj);
  const int64_t stride = static_cast<int64_t>(gridDim.x) * (GT * GT);
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int e = blockIdx.y * 1024 + q * 256 + threadIdx.x;
    const int m = e / GT, n = e % GT;
    const int i = bi * GT + m, j = bj * GT + n;
    if (i >= D || j >= D || (bi == bj && m > n)) continue;
    const double* p = part + static_cast<int64_t>(blockIdx.x) * (GT * GT) + e;
    double v = 0.0;
    for (int s = 0; s < S; ++s) v += p[s * stride];
    gram[static_cast<int64_t>(i) * D + j] += v;
    if (i != j) gram[static_cast<int64_t>(j) * D + i] += v;
  }
}

// grid (ceil(D / 32), P), block (32, 8): column j = 32 blockIdx.x + tx, rows of block p strided by 8 over ty, then
// the 8 row lanes in order -> part[p][j].
__global__ void __launch_bounds__(256) col_sum_part_kernel(const float* __restrict__ x, int64_t N, int D,
                                                           int64_t rows_per_part, double* __restrict__ part) {
  __shared__ double red[8][33];
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int j = blockIdx.x * 32 + tx;
  const int64_t r0 = static_cast<int64_t>(blockIdx.y) * rows_per_part;
  const int64_t r1 = min(N, r0 + rows_per_part);
  double s = 0.0;
  if (j < D) {
#pragma unroll 4
    for (int64_t r = r0 + ty; r < r1; r += 8) s += static_cast<double>(x[r * D + j]);
  }
  red[ty][tx] = s;
  __syncthreads();
  if (ty == 0 && j < D) {
    double v = red[0][tx];
#pragma unroll
    for (int w = 1; w < 8; ++w) v += red[w][tx];
    part[static_cast<int64_t>(blockIdx.y) * D + j] = v;
  }
}

__global__ void col_sum_reduce_kernel(const double* __restrict__ part, int P, int D, double* __restrict__ sum) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= D) return;
  double v = 0.0;
  for (int p = 0; p < P; ++p) v += part[static_cast<int64_t>(p) * D + j];
  sum[j] += v;
}

}  // namespace
}  // namespace dirb

using namespace dirb;

extern "C" {

int dirb200_col_sums_f64(const float* x_dev, int64_t N, int D, double* sum_dev, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DIRB_REQUIRE(N >= 0 && D > 0, DIRB200_EINVAL, "col_sums_f64: bad shape N %lld, D %d", (long long)N, D);
  DIRB_REQUIRE(sum_dev && (x_dev || N == 0), DIRB200_EINVAL, "col_sums_f64: null argument");
  DIRB_TRY(require_sm90());
  if (N == 0) return 0;
  const int64_t rows = std::max(CS_ROWS, ceil_div(N, CS_MAX_PARTS));
  const int P = static_cast<int>(ceil_div(N, rows));
  void* ws = nullptr;
  ScratchLease lease;
  DIRB_TRY(lease.acquire(static_cast<size_t>(P) * D * 8, stream, &ws));
  double* part = static_cast<double*>(ws);
  col_sum_part_kernel<<<dim3(static_cast<unsigned>(ceil_div(D, 32)), P), dim3(32, 8), 0, stream>>>(x_dev, N, D, rows, part);
  col_sum_reduce_kernel<<<static_cast<unsigned>(ceil_div(D, 256)), 256, 0, stream>>>(part, P, D, sum_dev);
  count_launch(2);
  DIRB_CUDA(cudaGetLastError());
  return 0;
}

int dirb200_gram_f64(const float* x_dev, int64_t N, int D, const double* mean_dev, double* gram_dev, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DIRB_REQUIRE(N >= 0 && D > 0, DIRB200_EINVAL, "gram_f64: bad shape N %lld, D %d", (long long)N, D);
  DIRB_REQUIRE(D % 4 == 0, DIRB200_EINVAL, "gram_f64: D must be a multiple of 4 (got %d)", D);
  DIRB_REQUIRE(mean_dev && gram_dev && (x_dev || N == 0), DIRB200_EINVAL, "gram_f64: null argument");
  DIRB_REQUIRE(D <= D_MAX, DIRB200_ENOTSUP,
               "gram_f64: D %d exceeds %d (the partial tiles of one split must fit the %d MiB workspace)", D, D_MAX,
               static_cast<int>(GRAM_WS_BYTES >> 20));
  DIRB_TRY(require_sm90());
  if (N == 0) return 0;
  const int T = static_cast<int>(ceil_div(D, GT));
  const int tiles = T * (T + 1) / 2;
  // splits: a function of (N, D) only - at least GRAM_SPLIT_ROWS rows each, all partials within GRAM_WS_BYTES
  const int64_t s_max = GRAM_MAX_TILES / tiles;
  const int64_t s_want = std::min<int64_t>(s_max, std::max<int64_t>(1, N / GRAM_SPLIT_ROWS));
  const int64_t rows = ceil_div(ceil_div(N, s_want), GK) * GK;
  const int S = static_cast<int>(ceil_div(N, rows));
  void* ws = nullptr;
  ScratchLease lease;
  DIRB_TRY(lease.acquire(static_cast<size_t>(S) * tiles * GRAM_TILE_BYTES, stream, &ws));
  double* part = static_cast<double*>(ws);
  static std::atomic<uint64_t> attr_done{0};
  if (first_launch_on_device(attr_done))
    DIRB_CUDA(cudaFuncSetAttribute(gram_tile_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, G_SMEM));
  gram_tile_kernel<<<dim3(tiles, S), G_THREADS, G_SMEM, stream>>>(x_dev, N, D, mean_dev, rows, T, part);
  gram_reduce_kernel<<<dim3(tiles, GT * GT / 1024), 256, 0, stream>>>(part, S, T, D, gram_dev);
  count_launch(2);
  DIRB_CUDA(cudaGetLastError());
  return 0;
}

}  // extern "C"
