// Fused stem for sm_90a: space-to-depth + 7x7/s2 convolution (3 -> 64) + BN + ReLU + 3x3/s2 max-pool in ONE persistent
// kernel that reads the images (NCHW fp32, or HWC uint8 normalised on the fly) and writes the pooled NHWC fp16 map.
//
// Tile: 7 x 7 pooled pixels of one image, which need the 15 x 15 stem pixels 2*py0-1 .. 2*py0+13 (and the same in x);
// the tile computes 16 x 16 stem pixels (two 8-pixel column panels, 16 rows), so neighbouring tiles recompute one stem
// row / column: 256 / 196 = 1.31x the MMA work of the stem.  Per tile:
//   1. all 256 threads write the 19 x 19 pixel space-to-depth patch S (16 fp16 channels per 2x2 input block, the
//      values of s2d_kernel / s2d_u8_kernel in conv.cu; uint8 bytes through a 3 x 256 table of their normalised
//      values) to shared memory, channel-chunk-major without swizzle:
//      [2 chunks of 8 channels][19][19][8] - K-major core matrices, as in the HALO mode of conv_pers.cuh;
//   2. warpgroup w computes stem rows 8w .. 8w+7 of both panels: the 16 taps (a, b) of the 4x4/s1 convolution over S
//      are 16 shifted wgmma descriptors into the patch (one k16 step each, a outer, b inner, the first without
//      accumulate: the K order of the unfused 4x1 convolution over the row-expanded tensor, so the bits are the same);
//      the weights W2 (64 x 256 fp16) stay in shared memory for the whole CTA;
//   3. epilogue fmaf(acc, scale, shift) -> ReLU -> fp16 into a 16 x 16 x 64 stem tile in shared memory;
//   4. the 3x3/s2 max over that tile (the order and -65504 start of maxpool_kernel, ops.cu) -> global memory.
// The global loads of the next tile's input are issued while the tensor cores run this tile's MMAs; two CTAs per SM
// overlap one tile's epilogue / pooling with the other's MMAs.
#pragma once
#include <type_traits>

#include "common.h"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace dirb {

constexpr int SP_PT = 7;                      // pooled pixels per tile side
constexpr int SP_T = 16;                      // stem pixels per tile side (2 * SP_PT + 1 used)
constexpr int SP_S = SP_T + 3;                // space-to-depth pixels per patch side
constexpr int SP_ITEMS = SP_S * SP_S;         // patch pixels
constexpr int SP_THREADS = 256;               // two warpgroups
constexpr int SP_ITEMS_PER_THREAD = (SP_ITEMS + SP_THREADS - 1) / SP_THREADS;
constexpr int SP_TP = 144;                    // bytes per stem-tile pixel: 64 fp16 channels + 16 bytes of padding, which
                                              // keeps the epilogue's stores and the pooling's 16-byte loads conflict-free

struct StemPoolSmem {
  static constexpr int W_OFF = 0;                        // W2 as [tap 16][chunk 2][co 64][8]: 2 KB per tap
  static constexpr int W_BYTES = 64 * 256 * 2;
  static constexpr int S_OFF = W_OFF + W_BYTES;
  static constexpr int S_CHUNK = SP_ITEMS * 16;          // one 8-channel chunk of the patch
  static constexpr int T_OFF = (S_OFF + 2 * S_CHUNK + 127) / 128 * 128;
  static constexpr int T_BYTES = SP_T * SP_T * SP_TP;    // stem tile [16][16] pixels of SP_TP bytes
  static constexpr int N_OFF = T_OFF + T_BYTES;          // uint8 input: normalised value of each byte, per channel
  static constexpr int TOTAL = N_OFF + 3 * 256 * 4;
};

struct StemPoolParams {
  const float* imgs;           // NCHW fp32 (B,3,H,W), or
  const uint8_t* imgs_u8;      // HWC uint8 (B,H,W,3) with
  float m0, m1, m2, s0, s1, s2;  // ... mean / std of the normalisation
  const __half* w2;            // [64][256] (pack_stem_w2)
  const float* scale;
  const float* shift;
  __half* out;                 // pooled map (B,Hp,Wp,64)
  __half* stem_out;            // optional: the stem map (B,Ho,Wo,64) before pooling (debug taps)
  int H, W, Ho, Wo, Hp, Wp;
  int tiles_x, tiles_y, total_tiles;
  // ragged batches: image n's {h, w} at level 0 (input), 1 (stem map), 2 (pooled map) at ext_l + n * ext_ld; null = dense
  const int* ext0;
  const int* ext1;
  const int* ext2;
  int ext_ld;
};

struct StemTile {
  int n, ty, tx, sy0, sx0;     // image, tile row / column, stem-map origin of the tile (= patch origin in S)
};
__device__ __forceinline__ StemTile stem_tile(const StemPoolParams& p, int t) {
  StemTile c;
  c.tx = t % p.tiles_x;
  c.ty = (t / p.tiles_x) % p.tiles_y;
  c.n = t / (p.tiles_x * p.tiles_y);
  c.sy0 = 2 * SP_PT * c.ty - 1;
  c.sx0 = 2 * SP_PT * c.tx - 1;
  return c;
}

// Raw input of one thread's patch pixels: 12 values (2x2 pixels x 3 channels) per pixel, loaded one tile ahead.
template <bool U8>
struct StemRaw {
  using T = typename std::conditional<U8, uint32_t, float>::type;
  T v[SP_ITEMS_PER_THREAD][12];
  uint32_t ok;                 // bit 4q + (dy*2+dx): the pixel lies inside the picture (else it enters as 0)
};

// S[Y][X][(dy*2+dx)*4 + c] = img[c][2Y+dy-3][2X+dx-3], masked by coordinate against the picture (s2d_kernel's rule).
template <bool U8>
__device__ __forceinline__ void stem_load(const StemPoolParams& p, const StemTile& c, StemRaw<U8>& r) {
  const unsigned hn = p.ext0 ? __ldg(p.ext0 + static_cast<int64_t>(c.n) * p.ext_ld) : p.H;
  const unsigned wn = p.ext0 ? __ldg(p.ext0 + static_cast<int64_t>(c.n) * p.ext_ld + 1) : p.W;
  const int64_t plane = static_cast<int64_t>(p.H) * p.W;
  const float* img = p.imgs + c.n * 3 * plane;                 // (the pointer of the other input type is unused)
  const uint8_t* img8 = p.imgs_u8 + c.n * 3 * plane;
  r.ok = 0;
#pragma unroll
  for (int q = 0; q < SP_ITEMS_PER_THREAD; ++q) {
    if (static_cast<int>(threadIdx.x & ~31u) + q * SP_THREADS >= SP_ITEMS) break;   // warp-uniform: no pixel left
    const int item = static_cast<int>(threadIdx.x) + q * SP_THREADS;
    const int Y = item / SP_S, X = item - (item / SP_S) * SP_S;
    const int y0 = 2 * (c.sy0 + Y) - 3, x0 = 2 * (c.sx0 + X) - 3;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int y = y0 + (k >> 1), x = x0 + (k & 1);
      const bool in = item < SP_ITEMS && static_cast<unsigned>(y) < hn && static_cast<unsigned>(x) < wn;
      r.ok |= (in ? 1u : 0u) << (4 * q + k);
      const int off = y * p.W + x;                              // 3 * H * W < 2^31 (stem_pool)
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) {
        if constexpr (U8) r.v[q][3 * k + ch] = in ? __ldg(img8 + off * 3 + ch) : 0u;
        else r.v[q][3 * k + ch] = in ? __ldg(img + ch * plane + off) : 0.f;
      }
    }
  }
}

template <bool U8>
__device__ __forceinline__ void stem_store_patch(const StemRaw<U8>& r, uint32_t s_addr, uint32_t n_addr) {
  using L = StemPoolSmem;
#pragma unroll
  for (int q = 0; q < SP_ITEMS_PER_THREAD; ++q) {
    if (static_cast<int>(threadIdx.x & ~31u) + q * SP_THREADS >= SP_ITEMS) break;   // warp-uniform: no pixel left
    const int item = static_cast<int>(threadIdx.x) + q * SP_THREADS;
    if (item >= SP_ITEMS) break;
    uint32_t o[8];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float c0 = 0.f, c1 = 0.f, c2 = 0.f;
      if ((r.ok >> (4 * q + k)) & 1u) {
        if constexpr (U8) {
          asm("ld.shared.f32 %0, [%1];" : "=f"(c0) : "r"(n_addr + r.v[q][3 * k] * 4));
          asm("ld.shared.f32 %0, [%1];" : "=f"(c1) : "r"(n_addr + 1024 + r.v[q][3 * k + 1] * 4));
          asm("ld.shared.f32 %0, [%1];" : "=f"(c2) : "r"(n_addr + 2048 + r.v[q][3 * k + 2] * 4));
        } else {
          c0 = r.v[q][3 * k];
          c1 = r.v[q][3 * k + 1];
          c2 = r.v[q][3 * k + 2];
        }
      }
      o[2 * k] = pack_h2(c0, c1);
      o[2 * k + 1] = pack_h2(c2, 0.f);
    }
    sts128(s_addr + item * 16, make_uint4(o[0], o[1], o[2], o[3]));
    sts128(s_addr + L::S_CHUNK + item * 16, make_uint4(o[4], o[5], o[6], o[7]));
  }
}

template <bool U8>
__global__ void __launch_bounds__(SP_THREADS, 2) stem_pool_kernel(const StemPoolParams p) {
  using L = StemPoolSmem;
  extern __shared__ __align__(128) uint8_t smem[];
  const uint32_t w_addr = smem_u32(smem) + L::W_OFF;
  const uint32_t s_addr = smem_u32(smem) + L::S_OFF;
  const uint32_t t_addr = smem_u32(smem) + L::T_OFF;
  const uint32_t n_addr = smem_u32(smem) + L::N_OFF;
  const int tid = threadIdx.x;
  const int wg = tid >> 7, wq = (tid >> 5) & 3, lane = tid & 31, g = lane >> 2, t4 = lane & 3;

  pdl_launch_dependents();   // the next kernel may start its own prologue while this one runs / drains
  pdl_wait();                // the images may come from the previous kernel of the stream

  // W2 row co = 32 vectors of 8 K values; vector v = tap (v / 2), chunk (v % 2).  No-swizzle K-major B operand:
  // the two chunks of a k16 step 1024 B apart (LBO), 8-channel groups 128 B apart (SBO).
  for (int i = tid; i < 64 * 32; i += SP_THREADS) {
    const int co = i >> 5, v = i & 31;
    sts128(w_addr + (v >> 1) * 2048 + (v & 1) * 1024 + co * 16, __ldg(reinterpret_cast<const uint4*>(p.w2) + i));
  }
  if constexpr (U8) {   // ToTensor + Normalize in fp32 with true divisions, as s2d_u8_kernel, once per byte value
    for (int i = tid; i < 3 * 256; i += SP_THREADS) {
      const int ch = i >> 8;
      const float m = ch == 0 ? p.m0 : ch == 1 ? p.m1 : p.m2, sd = ch == 0 ? p.s0 : ch == 1 ? p.s1 : p.s2;
      sts32f(n_addr + i * 4, __fdiv_rn(__fdiv_rn(static_cast<float>(i & 255), 255.0f) - m, sd));
    }
  }
  __syncthreads();

  float acc[2][32];
#pragma unroll
  for (int pn = 0; pn < 2; ++pn)
#pragma unroll
    for (int j = 0; j < 32; ++j) acc[pn][j] = 0.f;

  // wgmma descriptors of tap 0 (this warpgroup's first stem row, panel 0); the taps and panels add their byte offset / 16
  const uint64_t adesc0 = gmma_desc_noswizzle(s_addr + 8 * wg * SP_S * 16, L::S_CHUNK, SP_S * 16);
  const uint64_t bdesc0 = gmma_desc_noswizzle(w_addr, 1024, 128);

  StemRaw<U8> raw;
  int t = blockIdx.x;
  StemTile next = stem_tile(p, t);
  if (t < p.total_tiles) stem_load<U8>(p, next, raw);
  for (; t < p.total_tiles; t += gridDim.x) {
    const StemTile c = next;
    // the previous tile's MMAs have finished reading the patch (wgmma_wait below, then the barrier before pooling)
    stem_store_patch<U8>(raw, s_addr, n_addr);
    fence_proxy_async_smem();                       // generic-proxy smem writes -> visible to wgmma
    __syncthreads();                                // also: every thread is done pooling the previous stem tile

    // -------------------------------------------------------------- MMAs: 16 taps x 2 panels, K order a outer, b inner
#pragma unroll
    for (int pn = 0; pn < 2; ++pn)
#pragma unroll
      for (int j = 0; j < 32; ++j) fence_operand(acc[pn][j]);
    wgmma_fence();
#pragma unroll
    for (int tap = 0; tap < 16; ++tap) {
      const int a = tap >> 2, b = tap & 3;
#pragma unroll
      for (int pn = 0; pn < 2; ++pn) {
        // accumulator row r = 8 * gi + ri is stem pixel (8 wg + gi, 8 pn + ri): row gi + a, column 8 pn + ri + b of S
        wgmma_m64n64k16(acc[pn], adesc0 + (a * SP_S + 8 * pn + b), bdesc0 + tap * (2048 >> 4), tap != 0);
      }
    }
    wgmma_commit();
    if (t + static_cast<int>(gridDim.x) < p.total_tiles) {   // the next tile's input streams in under the MMAs
      next = stem_tile(p, t + gridDim.x);
      stem_load<U8>(p, next, raw);
    }
    wgmma_wait<0>();
#pragma unroll
    for (int pn = 0; pn < 2; ++pn)
#pragma unroll
      for (int j = 0; j < 32; ++j) fence_operand(acc[pn][j]);

    // -------------------------------------------------------------- epilogue -> stem tile in shared memory
    // Outside the picture's stem extent (ragged batches) the map is 0, as the unfused convolution epilogue writes it.
    const int eh1 = p.ext1 ? __ldg(p.ext1 + static_cast<int64_t>(c.n) * p.ext_ld) : p.Ho;
    const int ew1 = p.ext1 ? __ldg(p.ext1 + static_cast<int64_t>(c.n) * p.ext_ld + 1) : p.Wo;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int col = j * 8 + 2 * t4;
      const float2 sc = __ldg(reinterpret_cast<const float2*>(p.scale + col));
      const float2 sh = __ldg(reinterpret_cast<const float2*>(p.shift + col));
#pragma unroll
      for (int pn = 0; pn < 2; ++pn)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int ly = 8 * wg + 2 * wq + h, lx = 8 * pn + g;
          float v0 = fmaxf(fmaf(acc[pn][4 * j + 2 * h], sc.x, sh.x), 0.f);
          float v1 = fmaxf(fmaf(acc[pn][4 * j + 2 * h + 1], sc.y, sh.y), 0.f);
          if (c.sy0 + ly >= eh1 || c.sx0 + lx >= ew1) {
            v0 = 0.f;
            v1 = 0.f;
          }
          asm volatile("st.shared.u32 [%0], %1;" ::"r"(t_addr + (ly * SP_T + lx) * SP_TP + col * 2), "r"(pack_h2(v0, v1))
                       : "memory");
        }
    }
    __syncthreads();

    if (p.stem_out != nullptr) {   // debug taps: the stem pixels of the tile inside the map, 8 channels per store
      for (int i = tid; i < SP_T * SP_T * 8; i += SP_THREADS) {
        const int c8 = i & 7, ly = i >> 7, lx = (i >> 3) & (SP_T - 1);
        const int y = c.sy0 + ly, x = c.sx0 + lx;
        if (y >= 0 && y < p.Ho && x >= 0 && x < p.Wo)
          *reinterpret_cast<uint4*>(p.stem_out + ((static_cast<int64_t>(c.n) * p.Ho + y) * p.Wo + x) * 64 + c8 * 8) =
              lds128(t_addr + (ly * SP_T + lx) * SP_TP + c8 * 16);
      }
    }

    // -------------------------------------------------------------- 3x3/s2 max-pool, 8 channels per item
    const int eh2 = p.ext2 ? __ldg(p.ext2 + static_cast<int64_t>(c.n) * p.ext_ld) : p.Hp;
    const int ew2 = p.ext2 ? __ldg(p.ext2 + static_cast<int64_t>(c.n) * p.ext_ld + 1) : p.Wp;
    for (int i = tid; i < SP_PT * SP_PT * 8; i += SP_THREADS) {
      const int c8 = i & 7, pi = (i >> 3) / SP_PT, pj = (i >> 3) % SP_PT;
      const int py = SP_PT * c.ty + pi, px = SP_PT * c.tx + pj;
      if (py >= p.Hp || px >= p.Wp) continue;
      uint4 r = make_uint4(0u, 0u, 0u, 0u);
      if (py < eh2 && px < ew2) {
        __half2 m[4];
        const __half2 ninf = __floats2half2_rn(-65504.f, -65504.f);
#pragma unroll
        for (int e = 0; e < 4; ++e) m[e] = ninf;
        const uint32_t base = t_addr + (2 * pi * SP_T + 2 * pj) * SP_TP + c8 * 16;
        const int y0 = c.sy0 + 2 * pi, x0 = c.sx0 + 2 * pj;
#pragma unroll
        for (int dy = 0; dy < 3; ++dy) {
          if (static_cast<unsigned>(y0 + dy) >= static_cast<unsigned>(p.Ho)) continue;
#pragma unroll
          for (int dx = 0; dx < 3; ++dx) {
            if (static_cast<unsigned>(x0 + dx) >= static_cast<unsigned>(p.Wo)) continue;
            const uint4 v = lds128(base + (dy * SP_T + dx) * SP_TP);
            const __half2* hv = reinterpret_cast<const __half2*>(&v);
#pragma unroll
            for (int e = 0; e < 4; ++e) m[e] = __hmax2(m[e], hv[e]);
          }
        }
        r = *reinterpret_cast<uint4*>(m);
      }
      *reinterpret_cast<uint4*>(p.out + ((static_cast<int64_t>(c.n) * p.Hp + py) * p.Wp + px) * 64 + c8 * 8) = r;
    }
  }
}

}  // namespace dirb
