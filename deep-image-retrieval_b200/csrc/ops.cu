// Small memory-bound operators around the convolution stack and the descriptor post-processing.
// All of them are HBM-bound: one coalesced 16-byte access per thread per element group, fp32 arithmetic.
#include "conv.h"
#include "conv_pers.cuh"
#include "ptx.cuh"

#include <algorithm>
#include <mutex>

namespace dirb {

// ---------------------------------------------------------------------------------------------------------------
// NCHW fp32 (B,3,H,W) -> NHWC fp16 (B,H,W,8), channels 3..7 = 0.   (input staging for the stem, resnet.py:158)
__global__ void nchw_to_nhwc8_kernel(const float* __restrict__ in, __half* __restrict__ out, int64_t hw, int64_t total) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;  // pixel index over B*H*W
  if (i >= total) return;
  const int64_t b = i / hw, px = i - b * hw;
  const float* src = in + b * 3 * hw + px;
  uint4 o;
  o.x = pack_h2(src[0], src[hw]);
  o.y = pack_h2(src[2 * hw], 0.f);
  o.z = 0u;
  o.w = 0u;
  reinterpret_cast<uint4*>(out)[i] = o;
}

int nchw_to_nhwc8(const float* in, int B, int H, int W, __half* out, cudaStream_t stream) {
  const int64_t hw = static_cast<int64_t>(H) * W, total = hw * B;
  nchw_to_nhwc8_kernel<<<static_cast<unsigned>(ceil_div(total, 256)), 256, 0, stream>>>(in, out, hw, total);
  count_launch();
  DIRB_CUDA(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// MaxPool2d(kernel 3, stride 2, padding 1), NHWC fp16, 8 channels per thread.   (resnet.py:119,161)
// Ragged batch (ext != nullptr): outputs outside image b's extent are 0.  Inside, a window may reach beyond the
// extent into the zeros there: its inputs are >= 0 (after ReLU) and it holds a pixel of the image, so the maximum is
// the one of -inf padding.
__global__ void maxpool_kernel(const __half* __restrict__ in, __half* __restrict__ out, int B, int H, int W, int C,
                               int Ho, int Wo, const int* __restrict__ ext, int ext_ld) {
  const int cv = C / 8;
  const int64_t total = static_cast<int64_t>(B) * Ho * Wo * cv;
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= total) return;
  const int c8 = static_cast<int>(i % cv);
  int64_t r = i / cv;
  const int wo = static_cast<int>(r % Wo);
  r /= Wo;
  const int ho = static_cast<int>(r % Ho);
  const int b = static_cast<int>(r / Ho);
  __half2 m[4];
  const __half2 ninf = __floats2half2_rn(-65504.f, -65504.f);
#pragma unroll
  for (int e = 0; e < 4; ++e) m[e] = ninf;
#pragma unroll
  for (int dy = 0; dy < 3; ++dy) {
    const int hi = ho * 2 - 1 + dy;
    if (hi < 0 || hi >= H) continue;
#pragma unroll
    for (int dx = 0; dx < 3; ++dx) {
      const int wi = wo * 2 - 1 + dx;
      if (wi < 0 || wi >= W) continue;
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(in + ((static_cast<int64_t>(b) * H + hi) * W + wi) * C) + c8);
      const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
      for (int e = 0; e < 4; ++e) m[e] = __hmax2(m[e], h[e]);
    }
  }
  if (ext != nullptr && (ho >= __ldg(ext + static_cast<int64_t>(b) * ext_ld) || wo >= __ldg(ext + static_cast<int64_t>(b) * ext_ld + 1))) {
    reinterpret_cast<uint4*>(out)[i] = make_uint4(0u, 0u, 0u, 0u);
    return;
  }
  reinterpret_cast<uint4*>(out)[i] = *reinterpret_cast<uint4*>(m);
}

int maxpool_3x3s2(const __half* in, int B, int H, int W, int C, __half* out, cudaStream_t stream, const ConvExt* ext) {
  DIRB_REQUIRE(C % 8 == 0, DIRB200_ENOTSUP, "maxpool needs C %% 8 == 0");
  const int Ho = (H + 2 - 3) / 2 + 1, Wo = (W + 2 - 3) / 2 + 1;
  const int64_t total = static_cast<int64_t>(B) * Ho * Wo * (C / 8);
  maxpool_kernel<<<static_cast<unsigned>(ceil_div(total, 256)), 256, 0, stream>>>(in, out, B, H, W, C, Ho, Wo, ext ? ext->hw : nullptr,
                                                                               ext ? ext->ld : 0);
  count_launch();
  DIRB_CUDA(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// Head: global pooling (GeM / max / avg) -> (L2 over C) -> FC + bias -> L2.      (rmac_resnet.py:59-68, pooling.py:38-40)
// Four phases: 1 partial pooling (streams the NHWC feature map once - the only large read), 2 finish the pooling
// (+ optional L2 over channels), 3 FC + bias, 4 L2 (+ fp16 copy).  Every phase is written as the body of one "virtual
// block" (256 threads), used two ways with the SAME arithmetic in the same order, so the results are bit-identical:
//   * head_fused_kernel: ONE persistent launch, every CTA loops over the virtual blocks of a phase and the phases are
//     separated by a self-resetting grid barrier (default for the plain head);
//   * one kernel per phase (FPN head, which pools two maps side by side; option head_fused = 0).
// Buffers produced by one phase and consumed by the next (partial, g, y) are read with ld.global.cg / .ca, never
// through the non-coherent path: in the fused kernel they were written by other CTAs of the same launch.
namespace {

constexpr int HEAD_PX_LANES = 8;
constexpr int HEAD_THREADS = 256;

// Number of partial sums of one image's pooling: depends on its pixel count only, so that a descriptor does not depend
// on the batch it was computed in (the partial sums of one image are always combined in the same order).
__host__ __device__ __forceinline__ int head_splits_hw(int HW) { return max(1, min(16, HW / 64)); }

// Ragged batch: image b pools its own ext[b*ld] x ext[b*ld+1] pixels; pixel p of it sits at row p / w, column p % w
// of a map whose rows are slot_w pixels long.
struct HeadExt {
  const int* ext;
  int ld, slot_w;
};

__device__ __forceinline__ float gem_pow(float x, float p, int p_is3) { return p_is3 ? x * x * x : powf(x, p); }

struct HeadSmem {
  float red[HEAD_PX_LANES][256 + 8];
  float sh[32];
};

// phase 1, virtual grid (C/256, S, B): thread = (pixel lane 0..7, channel group 0..31 of 8 channels)
__device__ __forceinline__ void head_pool_partial_body(HeadSmem& sm, int bx, int s, int b, const __half* __restrict__ feat,
                                                       float* partial, int HW, int C, int S, int pooling, float p,
                                                       float eps, const HeadExt& he) {
  const int cg = threadIdx.x & 31, pl = threadIdx.x >> 5;
  const int c0 = bx * 256 + cg * 8;
  int hw = HW, Sb = S, wb = 1;
  if (he.ext != nullptr) {                                  // S = the slot's splits, Sb <= S of them are this image's
    wb = __ldg(he.ext + static_cast<int64_t>(b) * he.ld + 1);
    hw = __ldg(he.ext + static_cast<int64_t>(b) * he.ld) * wb;
    Sb = head_splits_hw(hw);
    if (s >= Sb) return;                                    // uniform over the (virtual) block
  }
  const int per = (hw + Sb - 1) / Sb;
  const int beg = s * per, end = min(hw, beg + per);
  const int p_is3 = (p == 3.0f);
  float acc[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) acc[e] = (pooling == 1) ? -INFINITY : 0.f;
  if (c0 < C) {
    for (int px = beg + pl; px < end; px += HEAD_PX_LANES) {
      const int64_t at = he.ext != nullptr ? static_cast<int64_t>(px / wb) * he.slot_w + px % wb : px;
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(feat + (static_cast<int64_t>(b) * HW + at) * C + c0));
      const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = unpack_h2(u[e]);
        if (pooling == 0) {
          acc[2 * e] += gem_pow(fmaxf(f.x, eps), p, p_is3);
          acc[2 * e + 1] += gem_pow(fmaxf(f.y, eps), p, p_is3);
        } else if (pooling == 1) {
          acc[2 * e] = fmaxf(acc[2 * e], f.x);
          acc[2 * e + 1] = fmaxf(acc[2 * e + 1], f.y);
        } else {
          acc[2 * e] += f.x;
          acc[2 * e + 1] += f.y;
        }
      }
    }
  }
#pragma unroll
  for (int e = 0; e < 8; ++e) sm.red[pl][cg * 8 + e] = acc[e];
  __syncthreads();
  const int c = threadIdx.x;
  if (bx * 256 + c < C) {
    float r = sm.red[0][c];
#pragma unroll
    for (int l = 1; l < HEAD_PX_LANES; ++l) r = (pooling == 1) ? fmaxf(r, sm.red[l][c]) : r + sm.red[l][c];
    partial[(static_cast<int64_t>(b) * S + s) * C + bx * 256 + c] = r;
  }
  __syncthreads();                                          // sm.red is free for the caller's next virtual block
}

__device__ __forceinline__ float block_sum(float v, float* sh) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = blockDim.x >> 5;
  __syncthreads();
  if (l == 0) sh[w] = v;
  __syncthreads();
  float t = (l < nw) ? sh[l] : 0.f;
  for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  return t;
}

// phase 2, one virtual block per image: finish the pooling, optional L2 over channels.  The pooled vector goes to
// columns [col_off, col_off + C) of row b of g (row length g_ld): two feature maps can be pooled side by side (FPN).
__device__ __forceinline__ void head_pool_final_body(HeadSmem& sm, int b, const float* partial, float* g, int HW, int C,
                                                     int S, int pooling, float p, int norm_features, int g_ld,
                                                     int col_off, const HeadExt& he) {
  float* grow = g + static_cast<int64_t>(b) * g_ld + col_off;
  float ss = 0.f;
  int Sb = S;
  if (he.ext != nullptr) {
    HW = __ldg(he.ext + static_cast<int64_t>(b) * he.ld) * __ldg(he.ext + static_cast<int64_t>(b) * he.ld + 1);
    Sb = head_splits_hw(HW);
  }
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float r = __ldcg(partial + (static_cast<int64_t>(b) * S) * C + c);
    for (int s = 1; s < Sb; ++s) {
      const float q = __ldcg(partial + (static_cast<int64_t>(b) * S + s) * C + c);
      r = (pooling == 1) ? fmaxf(r, q) : r + q;
    }
    if (pooling == 0) r = powf(r / static_cast<float>(HW), 1.0f / p);
    else if (pooling == 2) r = r / static_cast<float>(HW);
    grow[c] = r;
    ss += r * r;
  }
  if (norm_features) {
    const float tot = block_sum(ss, sm.sh);
    const float inv = 1.0f / fmaxf(sqrtf(tot), 1e-12f);
    for (int c = threadIdx.x; c < C; c += blockDim.x) grow[c] *= inv;
  }
}

// phase 3, virtual grid (ceil(out/8), ceil(B/8)): y[b][o] = sum_c W[o][c] g[b][c] + bias[o]; warp = one output row
__device__ __forceinline__ void head_fc_body(int bx, int by, const float* g, const float* __restrict__ w,
                                             const float* __restrict__ bias, float* y, int B, int C, int out_dim) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int o = bx * 8 + warp;
  const int b0 = by * 8;
  if (o >= out_dim) return;                                 // (no block-wide synchronisation in this phase)
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
  const float4* wr = reinterpret_cast<const float4*>(w + static_cast<int64_t>(o) * C);
  for (int c4 = lane; c4 < C / 4; c4 += 32) {
    const float4 wv = __ldg(wr + c4);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (b0 + i < B) {
        const float4 gv = __ldca(reinterpret_cast<const float4*>(g + static_cast<int64_t>(b0 + i) * C) + c4);
        acc[i] = fmaf(wv.x, gv.x, acc[i]);
        acc[i] = fmaf(wv.y, gv.y, acc[i]);
        acc[i] = fmaf(wv.z, gv.z, acc[i]);
        acc[i] = fmaf(wv.w, gv.w, acc[i]);
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    float v = acc[i];
    for (int s = 16; s > 0; s >>= 1) v += __shfl_xor_sync(0xffffffffu, v, s);
    if (lane == 0 && b0 + i < B) y[static_cast<int64_t>(b0 + i) * out_dim + o] = v + (bias ? __ldg(bias + o) : 0.f);
  }
}

// phase 4, one virtual block per row: out = x / max(||x||, eps)
__device__ __forceinline__ void l2_row_body(HeadSmem& sm, int64_t r, const float* x, float* out, __half* out16, int D,
                                            float eps) {
  const float* xr = x + r * D;
  float ss = 0.f;
  for (int c = threadIdx.x; c < D; c += blockDim.x) {
    const float v = __ldcg(xr + c);
    ss += v * v;
  }
  const float tot = block_sum(ss, sm.sh);
  const float nrm = sqrtf(tot);
  const float inv = 1.0f / (eps > 0.f ? fmaxf(nrm, eps) : nrm);
  for (int c = threadIdx.x; c < D; c += blockDim.x) {
    const float v = __ldcg(xr + c) * inv;
    if (out) out[r * D + c] = v;
    if (out16) out16[r * D + c] = __float2half_rn(v);
  }
}

__global__ void __launch_bounds__(HEAD_THREADS) head_pool_partial_kernel(const __half* __restrict__ feat, float* partial,
                                                                         int HW, int C, int S, int pooling, float p,
                                                                         float eps, const HeadExt he) {
  __shared__ HeadSmem sm;
  head_pool_partial_body(sm, blockIdx.x, blockIdx.y, blockIdx.z, feat, partial, HW, C, S, pooling, p, eps, he);
}
__global__ void __launch_bounds__(HEAD_THREADS) head_pool_final_kernel(const float* partial, float* g, int HW, int C, int S,
                                                                       int pooling, float p, int norm_features, int g_ld,
                                                                       int col_off, const HeadExt he) {
  __shared__ HeadSmem sm;
  head_pool_final_body(sm, blockIdx.x, partial, g, HW, C, S, pooling, p, norm_features, g_ld, col_off, he);
}
__global__ void __launch_bounds__(HEAD_THREADS) head_fc_kernel(const float* g, const float* __restrict__ w,
                                                               const float* __restrict__ bias, float* y, int B, int C,
                                                               int out_dim) {
  head_fc_body(blockIdx.x, blockIdx.y, g, w, bias, y, B, C, out_dim);
}
__global__ void __launch_bounds__(HEAD_THREADS) l2_rows_kernel(const float* x, float* out, __half* out16, int D, float eps) {
  __shared__ HeadSmem sm;
  l2_row_body(sm, blockIdx.x, x, out, out16, D, eps);
}

// Grid barrier of a persistent launch whose CTAs are all co-resident (the launcher sizes the grid from the occupancy
// calculator).  bar[0] = arrival counter, bar[1] = generation.  Self-resetting: the last arrival zeroes the counter and
// bumps the generation, so the words only have to be zero once, at allocation, and survive CUDA-graph replays.
__device__ __forceinline__ void grid_barrier(unsigned int* bar, unsigned int nblocks) {
  __syncthreads();
  if (threadIdx.x == 0) {
    volatile unsigned int* gen = bar + 1;
    const unsigned int g0 = *gen;                           // cannot advance before this CTA has arrived
    __threadfence();                                        // this CTA's writes (ordered by the bar.sync above) -> gpu scope
    if (atomicAdd(bar, 1u) == nblocks - 1u) {
      bar[0] = 0u;
      __threadfence();
      atomicAdd(bar + 1, 1u);
    } else {
      while (*gen == g0) __nanosleep(32);
    }
    __threadfence();
  }
  __syncthreads();
}

struct HeadFusedParams {
  const __half* feat;
  const float* fc_w;
  const float* fc_b;
  float* partial;
  float* g;
  float* y;
  float* desc;
  __half* desc16;
  unsigned int* bar;
  int B, HW, C, S, pooling, norm_features, out_dim;
  float p, eps;
  HeadExt he;
};

__global__ void __launch_bounds__(HEAD_THREADS, 4) head_fused_kernel(const HeadFusedParams q) {
  __shared__ HeadSmem sm;
  const int nb = gridDim.x;
  {  // ---- 1: partial pooling
    const int gx = (q.C + 255) / 256;
    const int total = gx * q.S * q.B;
    for (int v = blockIdx.x; v < total; v += nb)
      head_pool_partial_body(sm, v % gx, (v / gx) % q.S, v / (gx * q.S), q.feat, q.partial, q.HW, q.C, q.S, q.pooling, q.p, q.eps,
                             q.he);
  }
  grid_barrier(q.bar, nb);
  for (int b = blockIdx.x; b < q.B; b += nb)   // ---- 2: finish the pooling
    head_pool_final_body(sm, b, q.partial, q.g, q.HW, q.C, q.S, q.pooling, q.p, q.norm_features, q.C, 0, q.he);
  const float* pre = q.g;
  int D = q.C;
  if (q.fc_w != nullptr) {
    grid_barrier(q.bar, nb);
    const int gx = (q.out_dim + 7) / 8, gy = (q.B + 7) / 8;   // ---- 3: FC + bias
    for (int v = blockIdx.x; v < gx * gy; v += nb) head_fc_body(v % gx, v / gx, q.g, q.fc_w, q.fc_b, q.y, q.B, q.C, q.out_dim);
    pre = q.y;
    D = q.out_dim;
  }
  grid_barrier(q.bar, nb);
  for (int b = blockIdx.x; b < q.B; b += nb)   // ---- 4: L2 (+ fp16 copy)
    l2_row_body(sm, b, pre, q.desc, q.desc16, D, 1e-12f);
}

}  // namespace

static int head_splits(int B, int HW, int C) {
  (void)B; (void)C;
  return head_splits_hw(HW);
}

static HeadExt head_ext(const ConvExt* ext) {
  return ext != nullptr ? HeadExt{ext->hw, ext->ld, ext->slot_w} : HeadExt{nullptr, 0, 0};
}

static size_t align32(size_t floats) { return (floats + 31) / 32 * 32; }   // 128-byte lines: no line shared by two buffers

size_t head_partial_floats(int B, int HW, int C) { return align32(static_cast<size_t>(B) * head_splits(B, HW, C) * C); }

size_t head_workspace_floats(int B, int HW, int C, int out_dim) {
  return head_partial_floats(B, HW, C) + align32(static_cast<size_t>(B) * C) +
         align32(static_cast<size_t>(B) * (out_dim > C ? out_dim : C)) + 32;   // + barrier words of the fused kernel
}

// Global pooling of one NHWC map into g[b][col_off .. col_off + C) (rows of g_ld floats); `partial` = B * S * C floats.
int head_pool(const __half* feat, int B, int HW, int C, int pooling, float p, float eps, int norm_features, float* partial,
              float* g, int g_ld, int col_off, cudaStream_t stream, const ConvExt* ext) {
  DIRB_REQUIRE(C % 8 == 0 && C % 4 == 0, DIRB200_ENOTSUP, "head needs C %% 8 == 0");
  DIRB_REQUIRE(pooling >= 0 && pooling <= 2, DIRB200_EINVAL, "pooling mode %d", pooling);
  const int S = head_splits(B, HW, C);
  dim3 g1((unsigned)ceil_div(C, 256), (unsigned)S, (unsigned)B);
  head_pool_partial_kernel<<<g1, HEAD_THREADS, 0, stream>>>(feat, partial, HW, C, S, pooling, p, eps, head_ext(ext));
  head_pool_final_kernel<<<B, HEAD_THREADS, 0, stream>>>(partial, g, HW, C, S, pooling, p, norm_features, g_ld, col_off,
                                                         head_ext(ext));
  count_launch(2);
  DIRB_CUDA(cudaGetLastError());
  return 0;
}

// Pooled features g [B][C] -> (fc + bias) -> L2 -> desc [B][D] (+ fp16 copy); y = B * out_dim floats of scratch.
int head_fc_l2(const float* g, int B, int C, const float* fc_w, const float* fc_b, int out_dim, float* y, float* desc,
               __half* desc16, cudaStream_t stream) {
  DIRB_REQUIRE(C % 4 == 0, DIRB200_ENOTSUP, "head needs C %% 4 == 0");
  const float* pre = g;
  int D = C;
  if (fc_w != nullptr) {
    dim3 g3((unsigned)ceil_div(out_dim, 8), (unsigned)ceil_div(B, 8));
    head_fc_kernel<<<g3, HEAD_THREADS, 0, stream>>>(g, fc_w, fc_b, y, B, C, out_dim);
    count_launch();
    pre = y;
    D = out_dim;
  }
  l2_rows_kernel<<<B, HEAD_THREADS, 0, stream>>>(pre, desc, desc16, D, 1e-12f);
  count_launch();
  DIRB_CUDA(cudaGetLastError());
  return 0;
}

static int g_head_fused = 1;   // tuning knob (option "head_fused"): 0 = one kernel per phase
void set_head_fused(int on) { g_head_fused = on; }
int get_head_fused() { return g_head_fused; }

// `bar`: two zero-initialised device words owned by the caller for the fused kernel's grid barrier (they return to a
// reusable state after every launch); nullptr = use the tail of `ws` and clear it on the stream first.
int head_pool_fc_l2(const __half* feat, int B, int HW, int C, int pooling, float p, float eps, int norm_features,
                    const float* fc_w, const float* fc_b, int out_dim, float* ws, float* desc, __half* desc16,
                    cudaStream_t stream, unsigned int* bar, const ConvExt* ext) {
  const int S = head_splits(B, HW, C);
  float* partial = ws;
  float* g = partial + head_partial_floats(B, HW, C);
  float* y = g + align32(static_cast<size_t>(B) * C);
  if (!g_head_fused) {
    DIRB_TRY(head_pool(feat, B, HW, C, pooling, p, eps, norm_features, partial, g, C, 0, stream, ext));
    return head_fc_l2(g, B, C, fc_w, fc_b, out_dim, y, desc, desc16, stream);
  }
  DIRB_REQUIRE(C % 8 == 0, DIRB200_ENOTSUP, "head needs C %% 8 == 0");
  DIRB_REQUIRE(pooling >= 0 && pooling <= 2, DIRB200_EINVAL, "pooling mode %d", pooling);
  if (bar == nullptr) {
    bar = reinterpret_cast<unsigned int*>(y + align32(static_cast<size_t>(B) * (out_dim > C ? out_dim : C)));
    DIRB_CUDA(cudaMemsetAsync(bar, 0, 2 * sizeof(unsigned int), stream));
  }
  // every CTA must be resident at once (spin barrier): grid = what the occupancy calculator guarantees, capped by the work
  static int per_sm = 0;
  if (per_sm == 0) {
    DIRB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, head_fused_kernel, HEAD_THREADS, 0));
    per_sm = std::max(1, std::min(per_sm, 4));
  }
  const int64_t work = std::max<int64_t>(ceil_div(C, 256) * S * B, fc_w ? ceil_div(out_dim, 8) * ceil_div(B, 8) : B);
  const int grid = static_cast<int>(std::min<int64_t>(static_cast<int64_t>(per_sm) * num_sms(), std::max<int64_t>(work, 1)));
  HeadFusedParams q{feat, fc_w, fc_b, partial, g, y, desc, desc16, bar, B, HW, C, S, pooling, norm_features, out_dim, p, eps,
                    head_ext(ext)};
  head_fused_kernel<<<grid, HEAD_THREADS, 0, stream>>>(q);
  count_launch();
  DIRB_CUDA(cudaGetLastError());
  return 0;
}

// FPN lateral connection (rmac_resnet_fpn.py:56-60): x4[b][y][x][:] += t[b][sy][sx][:], (sy, sx) = nearest-neighbour
// source of (y, x) as F.interpolate(mode='nearest', size=(H,W)) picks it: min(floor(dst * in / out), in - 1) with the
// ratio in fp32.  t is the 1x1-reduced, ReLU-ed layer4 map: the 1x1 convolution commutes with the upsampling, so it
// runs on the small map.  out may alias x4.  8 channels per thread.
__global__ void upsample_add_kernel(const __half* __restrict__ x4, const __half* __restrict__ t, __half* __restrict__ out,
                                    int H, int W, int h, int w, int C8, float sy, float sx, int64_t total) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c8 = static_cast<int>(i % C8);
  int64_t r = i / C8;
  const int x = static_cast<int>(r % W);
  r /= W;
  const int y = static_cast<int>(r % H);
  const int64_t b = r / H;
  const int yy = min(static_cast<int>(floorf(static_cast<float>(y) * sy)), h - 1);
  const int xx = min(static_cast<int>(floorf(static_cast<float>(x) * sx)), w - 1);
  const uint4 a = __ldg(reinterpret_cast<const uint4*>(x4) + i);
  const uint4 bv = __ldg(reinterpret_cast<const uint4*>(t) + ((b * h + yy) * w + xx) * C8 + c8);
  const __half2* ha = reinterpret_cast<const __half2*>(&a);
  const __half2* hb = reinterpret_cast<const __half2*>(&bv);
  uint4 o;
  __half2* ho = reinterpret_cast<__half2*>(&o);
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const float2 fa = __half22float2(ha[e]), fb = __half22float2(hb[e]);
    ho[e] = __floats2half2_rn(fa.x + fb.x, fa.y + fb.y);
  }
  reinterpret_cast<uint4*>(out)[i] = o;
}

int upsample_add(const __half* x4, const __half* t, __half* out, int B, int H, int W, int h, int w, int C,
                 cudaStream_t stream) {
  DIRB_REQUIRE(C % 8 == 0, DIRB200_ENOTSUP, "upsample_add needs C %% 8 == 0 (got %d)", C);
  const int64_t total = static_cast<int64_t>(B) * H * W * (C / 8);
  if (total == 0) return 0;
  upsample_add_kernel<<<static_cast<unsigned>(ceil_div(total, 256)), 256, 0, stream>>>(
      x4, t, out, H, W, h, w, C / 8, static_cast<float>(h) / static_cast<float>(H), static_cast<float>(w) / static_cast<float>(W), total);
  count_launch();
  DIRB_CUDA(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// center_bias (rmac_resnet.py:52-56): x[n][h][w][:] *= 1 + bilinear(align_corners=True) of the 4x4 map that is b on
// its central 2x2 and 0 on its border, resized to (H, W).  In place on the fp16 NHWC layer4 map, 8 channels / thread.
__device__ __forceinline__ float center_bias_axis(int i, int n, int& i0, int& i1, float& l1) {
  const float scale = n > 1 ? 3.0f / static_cast<float>(n - 1) : 0.0f;   // (in - 1) / (out - 1), in = 4
  const float src = scale * static_cast<float>(i);
  i0 = static_cast<int>(src);
  i1 = i0 + (i0 < 3 ? 1 : 0);
  l1 = src - static_cast<float>(i0);
  return 1.0f - l1;
}

// Ragged batch (ext != nullptr): the map is resized to image n's own extent; pixels outside it stay 0.
__global__ void center_bias_kernel(__half* __restrict__ x, int H, int W, int C8, float b, int64_t total,
                                   const int* __restrict__ ext, int ext_ld) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int64_t pix = i / C8;
  const int wq = static_cast<int>(pix % W);
  const int hq = static_cast<int>((pix / W) % H);
  if (ext != nullptr) {
    const int64_t n = pix / (static_cast<int64_t>(W) * H);
    H = __ldg(ext + n * ext_ld);
    W = __ldg(ext + n * ext_ld + 1);
    if (hq >= H || wq >= W) return;
  }
  int h0, h1, w0, w1;
  float lh1, lw1;
  const float lh0 = center_bias_axis(hq, H, h0, h1, lh1);
  const float lw0 = center_bias_axis(wq, W, w0, w1, lw1);
  auto tab = [b](int r, int c) { return (r == 1 || r == 2) && (c == 1 || c == 2) ? b : 0.0f; };
  const float m = 1.0f + (lh0 * (lw0 * tab(h0, w0) + lw1 * tab(h0, w1)) + lh1 * (lw0 * tab(h1, w0) + lw1 * tab(h1, w1)));
  uint4* ptr = reinterpret_cast<uint4*>(x) + i;
  uint4 v = *ptr;
  __half2* hv = reinterpret_cast<__half2*>(&v);
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    float2 f = __half22float2(hv[e]);
    f.x *= m;
    f.y *= m;
    hv[e] = __floats2half2_rn(f.x, f.y);
  }
  *ptr = v;
}

int center_bias(__half* x, int B, int H, int W, int C, float b, cudaStream_t stream, const ConvExt* ext) {
  DIRB_REQUIRE(C % 8 == 0, DIRB200_ENOTSUP, "center_bias needs C %% 8 == 0 (got %d)", C);
  const int64_t total = static_cast<int64_t>(B) * H * W * (C / 8);
  if (total == 0 || b == 0.0f) return 0;
  center_bias_kernel<<<static_cast<unsigned>(ceil_div(total, 256)), 256, 0, stream>>>(x, H, W, C / 8, b, total, ext ? ext->hw : nullptr,
                                                                                          ext ? ext->ld : 0);
  count_launch();
  DIRB_CUDA(cudaGetLastError());
  return 0;
}

int l2_normalize(const float* x, int64_t N, int D, float eps, float* out, __half* out16, cudaStream_t stream) {
  if (N == 0) return 0;
  l2_rows_kernel<<<static_cast<unsigned>(N), 256, 0, stream>>>(x, out, out16, D, eps);
  count_launch();
  DIRB_CUDA(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// common.pool over S transform chains (+ F.normalize): common.py:41-55, test_dir.py:121-122.
__global__ void pool_scales_kernel(const float* __restrict__ xs, float* __restrict__ out, int S, int64_t N, int D,
                                   int mode, float gemp, int l2) {
  __shared__ float sh[32];
  const int64_t r = blockIdx.x;
  float ss = 0.f;
  for (int c = threadIdx.x; c < D; c += blockDim.x) {
    float acc = 0.f;
    for (int s = 0; s < S; ++s) {
      const float v = xs[(static_cast<int64_t>(s) * N + r) * D + c];
      if (mode == 0) {
        acc += v;
      } else {  // signed power: sign(v) * max(|v|, 1e-6)^p
        const float sg = (v > 0.f) ? 1.f : ((v < 0.f) ? -1.f : 0.f);
        acc += sg * powf(fmaxf(v * sg, 1e-6f), gemp);
      }
    }
    acc /= static_cast<float>(S);
    if (mode == 1) {
      const float sg = (acc > 0.f) ? 1.f : ((acc < 0.f) ? -1.f : 0.f);
      acc = sg * powf(fmaxf(acc * sg, 1e-6f), 1.0f / gemp);
    }
    out[r * D + c] = acc;
    ss += acc * acc;
  }
  if (l2) {
    const float tot = block_sum(ss, sh);
    const float inv = 1.0f / fmaxf(sqrtf(tot), 1e-12f);
    for (int c = threadIdx.x; c < D; c += blockDim.x) out[r * D + c] *= inv;
  }
}

int pool_scales(const float* xs, int S, int64_t N, int D, int mode, float gemp, int l2, float* out,
                cudaStream_t stream) {
  DIRB_REQUIRE(S >= 1 && (mode == 0 || mode == 1), DIRB200_EINVAL, "pool_scales: S=%d mode=%d", S, mode);
  if (N == 0) return 0;
  if (S == 1) mode = 0;  // common.py:42-43: a single chain is returned unchanged
  pool_scales_kernel<<<static_cast<unsigned>(N), 256, 0, stream>>>(xs, out, S, N, D, mode, gemp, l2);
  count_launch();
  DIRB_CUDA(cudaGetLastError());
  return 0;
}

__global__ void f32_to_f16_kernel(const float* __restrict__ x, __half* __restrict__ out, int64_t n) {
  const int64_t i = (blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) * 4;
  if (i + 3 < n) {
    const float4 v = *reinterpret_cast<const float4*>(x + i);
    uint2 o;
    o.x = pack_h2(v.x, v.y);
    o.y = pack_h2(v.z, v.w);
    *reinterpret_cast<uint2*>(out + i) = o;
  } else {
    for (int64_t j = i; j < n; ++j) out[j] = __float2half_rn(x[j]);
  }
}

int f32_to_f16(const float* x, int64_t n, __half* out, cudaStream_t stream) {
  if (n == 0) return 0;
  f32_to_f16_kernel<<<static_cast<unsigned>(ceil_div(ceil_div(n, 4), 256)), 256, 0, stream>>>(x, out, n);
  count_launch();
  DIRB_CUDA(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// PCA whitening: Y = ((X - mean) . comp^T) * colscale, optional row L2.                     (common.py:221-239)
// fp32 SIMT GEMM, 64x64 tile, 4x4 per thread: exact fp32 products (the reference runs this in NumPy fp32/fp64).
namespace {
constexpr int WT = 64, WK = 16;

__global__ void __launch_bounds__(256) whiten_gemm_kernel(const float* __restrict__ x, const float* __restrict__ comp,
                                                          const float* __restrict__ mean,
                                                          const float* __restrict__ colscale, float* __restrict__ y,
                                                          int64_t N, int D, int Dout) {
  __shared__ float As[WK][WT + 4];
  __shared__ float Bs[WK][WT + 4];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int64_t m0 = static_cast<int64_t>(blockIdx.x) * WT;
  const int n0 = blockIdx.y * WT;
  const int lr = threadIdx.x >> 2, lk = (threadIdx.x & 3) * 4;  // loader: row 0..63, k offset 0,4,8,12
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int k0 = 0; k0 < D; k0 += WK) {
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;
    if (m0 + lr < N) {
      a = *reinterpret_cast<const float4*>(x + (m0 + lr) * D + k0 + lk);
      if (mean) {
        const float4 mu = *reinterpret_cast<const float4*>(mean + k0 + lk);
        a.x -= mu.x; a.y -= mu.y; a.z -= mu.z; a.w -= mu.w;
      }
    }
    if (n0 + lr < Dout) b = *reinterpret_cast<const float4*>(comp + static_cast<int64_t>(n0 + lr) * D + k0 + lk);
    __syncthreads();
    As[lk + 0][lr] = a.x; As[lk + 1][lr] = a.y; As[lk + 2][lr] = a.z; As[lk + 3][lr] = a.w;
    Bs[lk + 0][lr] = b.x; Bs[lk + 1][lr] = b.y; Bs[lk + 2][lr] = b.z; Bs[lk + 3][lr] = b.w;
    __syncthreads();
#pragma unroll
    for (int k = 0; k < WK; ++k) {
      float av[4], bv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) av[i] = As[k][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) bv[j] = Bs[k][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int64_t m = m0 + ty * 4 + i;
    if (m >= N) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n < Dout) y[m * Dout + n] = acc[i][j] * (colscale ? colscale[n] : 1.0f);
    }
  }
}
}  // namespace

// ---- device scratch cache -------------------------------------------------------------------------------------
// dirb200_whiten has no handle, and allocating ~1 GB of split buffers per call (cudaMallocAsync after every
// synchronisation point, i.e. a driver-level allocation) serialises badly when 8 processes share a box.  One scratch
// buffer per device is therefore kept for the life of the process (grown on demand).  Users on different streams are
// ordered through an event: acquire makes the caller's stream wait for the previous user, and the lease records the
// event once its work is enqueued.  The device's mutex is held for the whole lease, so a second caller cannot acquire
// between the first one's acquire and its record (it would wait on an older event and share the buffer).
namespace {
struct DevScratch {
  void* ptr = nullptr;
  size_t bytes = 0;
  cudaEvent_t last_use = nullptr;
  std::mutex mu;
};
DevScratch g_scratch[64];
}  // namespace

int ScratchLease::acquire(size_t bytes, cudaStream_t stream, void** out) {
  int dev = 0;
  DIRB_CUDA(cudaGetDevice(&dev));
  DIRB_REQUIRE(dev >= 0 && dev < 64, DIRB200_ENOTSUP, "device index %d out of range", dev);
  DIRB_REQUIRE(!lock_.owns_lock(), DIRB200_ESTATE, "scratch lease acquired twice");
  DevScratch& s = g_scratch[dev];
  lock_ = std::unique_lock<std::mutex>(s.mu);
  if (!s.last_use) DIRB_CUDA(cudaEventCreateWithFlags(&s.last_use, cudaEventDisableTiming));
  if (bytes > s.bytes) {
    // cudaFree synchronises the device: no earlier user is still running
    DIRB_TRY(grow_device(&s.ptr, &s.bytes, (bytes + (size_t(1) << 20) - 1) & ~((size_t(1) << 20) - 1)));
  } else {
    DIRB_CUDA(cudaStreamWaitEvent(stream, s.last_use, 0));
  }
  last_use_ = s.last_use;
  stream_ = stream;
  *out = s.ptr;
  return 0;
}

ScratchLease::~ScratchLease() {
  // the next lease's stream waits for everything this one enqueued (a destructor has no status to return: the record
  // fails only when the context is already broken, which the caller's next CUDA call reports)
  if (lock_.owns_lock() && last_use_) cudaEventRecord(last_use_, stream_);
}

// ---- fp16 hi/lo split with an adaptive power-of-two prescale --------------------------------------------------------
// v = x - mean is written as hi + lo (two fp16 numbers; hi + lo reproduces v to ~2^-22 relative).  The LOW half is
// ~ v * 2^-11: without a prescale it falls into fp16's subnormal range (< 6.1e-5, quantum 6e-8) as soon as |v| < ~0.1
// and the scheme degrades towards a single fp16 pass (relative error ~ 1 / |x - mean|, tests/test_properties.py).  Both
// operands are therefore multiplied by a power of two chosen from their largest magnitude (exact in fp32) so that
// max |v| lands in [2^13, 2^14): the low halves of all values within 2^-12 of the maximum stay normal; the product of
// the two scales is divided out in the column scale.
//   ws[0] = bits of max |x - mean|, ws[1] = bits of max |comp|   (atomicMax on the bit pattern: values are >= 0)
//   ws[2] = scale_x, ws[3] = scale_c, ws[4] = 1 / (scale_x * scale_c)
__global__ void absmax_kernel(const float* __restrict__ x, const float* __restrict__ mean, int D, int64_t total,
                              unsigned int* __restrict__ out_bits) {
  float m = 0.f;
  for (int64_t i = (blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) * 4; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x * 4) {
    float4 v = *reinterpret_cast<const float4*>(x + i);
    if (mean) {
      const float4 mu = *reinterpret_cast<const float4*>(mean + (i % D));
      v.x -= mu.x; v.y -= mu.y; v.z -= mu.z; v.w -= mu.w;
    }
    m = fmaxf(fmaxf(m, fmaxf(fabsf(v.x), fabsf(v.y))), fmaxf(fabsf(v.z), fabsf(v.w)));
  }
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m > 0.f && m < INFINITY) atomicMax(out_bits, __float_as_uint(m));
}

__device__ __forceinline__ float prescale_for(float absmax) {
  if (!(absmax > 0.f)) return 1.0f;
  int e;
  frexpf(absmax, &e);                       // absmax = f * 2^e, f in [0.5, 1)
  int sh = 14 - e;                          // absmax * 2^sh in [2^13, 2^14)
  sh = sh > 40 ? 40 : (sh < -40 ? -40 : sh);
  return ldexpf(1.0f, sh);
}

// ws[2..4] from ws[0..1]; cs[j] = (colscale ? colscale[j] : 1) / (scale_x * scale_c)
__global__ void pick_prescale_kernel(float* __restrict__ ws, const float* __restrict__ colscale, float* __restrict__ cs,
                                     int n) {
  const float sx = prescale_for(__uint_as_float(reinterpret_cast<unsigned int*>(ws)[0]));
  const float sc = prescale_for(__uint_as_float(reinterpret_cast<unsigned int*>(ws)[1]));
  const float inv = 1.0f / (sx * sc);
  if (threadIdx.x == 0) {
    ws[2] = sx;
    ws[3] = sc;
    ws[4] = inv;
  }
  for (int j = threadIdx.x; j < n; j += blockDim.x) cs[j] = (colscale ? colscale[j] : 1.0f) * inv;
}

__global__ void split_f16_kernel(const float* __restrict__ x, const float* __restrict__ mean, int D, int64_t total,
                                 const float* __restrict__ scale_ptr, __half* __restrict__ hi, __half* __restrict__ lo) {
  const int64_t i = (blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) * 4;
  if (i >= total) return;
  const float sc = *scale_ptr;
  float4 v = *reinterpret_cast<const float4*>(x + i);
  if (mean) {
    const float4 m = *reinterpret_cast<const float4*>(mean + (i % D));
    v.x -= m.x; v.y -= m.y; v.z -= m.z; v.w -= m.w;
  }
  v.x *= sc; v.y *= sc; v.z *= sc; v.w *= sc;               // power of two: exact
  const __half h0 = __float2half_rn(v.x), h1 = __float2half_rn(v.y), h2 = __float2half_rn(v.z), h3 = __float2half_rn(v.w);
  uint2 oh, ol;
  oh.x = pack_h2(__half2float(h0), __half2float(h1));
  oh.y = pack_h2(__half2float(h2), __half2float(h3));
  ol.x = pack_h2(v.x - __half2float(h0), v.y - __half2float(h1));
  ol.y = pack_h2(v.z - __half2float(h2), v.w - __half2float(h3));
  *reinterpret_cast<uint2*>(hi + i) = oh;
  *reinterpret_cast<uint2*>(lo + i) = ol;
}

// Tensor-core whitening: Y = ((X - mean) . comp^T) * colscale through three fp16 GEMM passes over hi/lo splits
// (hi*hi + hi*lo + lo*hi, fp32 accumulation in registers) - fp32-level accuracy at tensor-core speed.
static int whiten_tc(const float* x, int64_t N, int D, const float* comp, const float* mean, const float* colscale,
                     int Dout, float* y, cudaStream_t stream) {
  const size_t xe = static_cast<size_t>(N) * D, ce = static_cast<size_t>(Dout) * D;
  __half *xh, *xl, *ch, *cl;
  float *ws, *cs;
  auto layout = [&](void* base) {
    Carver c(base, 1024);
    xh = c.take<__half>(xe);
    xl = c.take<__half>(xe);
    ch = c.take<__half>(ce);
    cl = c.take<__half>(ce);
    ws = c.take<float>(256);
    cs = c.take<float>(Dout);
    return c.used;
  };
  void* base = nullptr;
  ScratchLease lease;
  DIRB_TRY(lease.acquire(layout(nullptr), stream, &base));
  layout(base);
  DIRB_CUDA(cudaMemsetAsync(ws, 0, 32, stream));
  const unsigned gx = static_cast<unsigned>(std::min<int64_t>(ceil_div(ceil_div(xe, 4), 256), num_sms() * 16));
  const unsigned gc = static_cast<unsigned>(std::min<int64_t>(ceil_div(ceil_div(ce, 4), 256), num_sms() * 16));
  absmax_kernel<<<gx, 256, 0, stream>>>(x, mean, D, xe, reinterpret_cast<unsigned int*>(ws));
  absmax_kernel<<<gc, 256, 0, stream>>>(comp, nullptr, D, ce, reinterpret_cast<unsigned int*>(ws) + 1);
  pick_prescale_kernel<<<1, 256, 0, stream>>>(ws, colscale, cs, Dout);
  split_f16_kernel<<<static_cast<unsigned>(ceil_div(ceil_div(xe, 4), 256)), 256, 0, stream>>>(x, mean, D, xe, ws + 2, xh, xl);
  split_f16_kernel<<<static_cast<unsigned>(ceil_div(ceil_div(ce, 4), 256)), 256, 0, stream>>>(comp, nullptr, D, ce, ws + 3, ch, cl);
  count_launch(5);
  DIRB_CUDA(cudaGetLastError());
  constexpr int BN = 128;
  CUtensorMap tmAh, tmAl, tmBh, tmBl;
  DIRB_TRY(encode_tmap_2d(&tmAh, xh, D, N, (uint64_t)D * 2, 64, 128));
  DIRB_TRY(encode_tmap_2d(&tmAl, xl, D, N, (uint64_t)D * 2, 64, 128));
  DIRB_TRY(encode_tmap_2d(&tmBh, ch, D, Dout, (uint64_t)D * 2, 64, BN));
  DIRB_TRY(encode_tmap_2d(&tmBl, cl, D, Dout, (uint64_t)D * 2, 64, BN));
  ConvPersParams p{};
  p.a_spatial = 0;
  p.taps = 1; p.kw_taps = 1;
  p.k_per_part = D / 64;
  p.cin_blocks = 3 * p.k_per_part;
  p.stride = 1; p.pad = 0;
  p.tw = 128; p.th = 1; p.nb = 1; p.tiles_w = 1; p.tiles_h = 1;
  p.M = static_cast<int>(N);
  p.N = Dout;
  p.n_tiles = static_cast<int>(ceil_div(Dout, BN));
  p.m_tiles = static_cast<int>(ceil_div(N, 128));
  p.m_fastest = 0;
  const int64_t total = static_cast<int64_t>(p.m_tiles) * p.n_tiles;
  DIRB_REQUIRE(total < (int64_t(1) << 31) && N < (int64_t(1) << 31), DIRB200_ENOTSUP, "whiten: shape too large");
  p.total_tiles = static_cast<int>(total);
  p.dense = y;
  p.dense_ld = Dout;
  p.scale = cs;
  return conv_pers_launch<BN, 6, PERS_EPI_F32>(tmAh, tmBh, tmAl, tmBl, p, num_sms(), stream);
}

int whiten(const float* x, int64_t N, int D, const float* comp, const float* mean, const float* colscale, int Dout,
           int l2norm, float* y, __half* y16, cudaStream_t stream) {
  DIRB_REQUIRE(D % WK == 0, DIRB200_ENOTSUP, "whiten needs D %% 16 == 0 (got %d)", D);
  if (N == 0) return 0;
  if (D % 64 == 0 && N >= 64) {
    DIRB_TRY(whiten_tc(x, N, D, comp, mean, colscale, Dout, y, stream));
  } else {
    dim3 grid((unsigned)ceil_div(N, WT), (unsigned)ceil_div(Dout, WT));
    DIRB_REQUIRE(ceil_div(N, WT) < (int64_t(1) << 31) && grid.y < 65536u, DIRB200_ENOTSUP, "whiten: shape too large");
    whiten_gemm_kernel<<<grid, 256, 0, stream>>>(x, comp, mean, colscale, y, N, D, Dout);
    count_launch();
    DIRB_CUDA(cudaGetLastError());
  }
  if (l2norm) return l2_normalize(y, N, Dout, 0.f, y, y16, stream);
  if (y16) return f32_to_f16(y, N * Dout, y16, stream);
  return 0;
}

}  // namespace dirb
