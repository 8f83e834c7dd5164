// Bottleneck tail in one persistent wgmma kernel for sm_90a: conv2 (3x3/s1/p1, Cm -> Cm) + BN + ReLU, then conv3
// (1x1, Cm -> 4 Cm) + BN + residual + ReLU, per 8 x 16-pixel tile (resnet.py:75-85).
//
//   warpgroup 0     TMA producer (one thread): per tile, conv2's input patches (one 5-D box per 64-channel block, as in
//                   the HALO mode of conv_pers.cuh) and its weight tiles, then conv3's weight tiles, into one ring
//   warpgroups 1-2  consumers, 64 pixel rows each.  conv2 runs in chunks of up to 128 output channels; its epilogue
//                   (BN, ReLU, fp16) writes the chunk into the tile's T2 buffer in shared memory, 128-byte swizzled,
//                   which is exactly the K-major A operand of conv3.  conv3 runs in chunks of 128 output channels with
//                   the epilogue of conv_pers.cuh (residual TMA-loaded into the staging buffers, TMA store).
//
// The conv2 output never goes to HBM.  K orders (channel block, then tap; fp32 accumulation) and epilogue arithmetic
// are those of conv_pers_kernel, so the result equals the two-kernel path bit for bit.  A warpgroup's conv3 reads only
// the T2 rows it wrote itself, so T2 needs no CTA-wide barrier.
#pragma once
#include "conv_pers.cuh"

namespace dirb {

template <int CM>
struct C23Smem {
  static constexpr int NB2 = CM < 128 ? CM : 128;                    // conv2 output channels per chunk
  static constexpr int STAGES = 4;
  static constexpr int SLOT = 128 * 128;                             // weight tile, up to 128 rows x 64 channels
  static constexpr int T2_BYTES = (CM / 64) * 128 * 128;
  static constexpr int PATCH_DATA = HALO_W * HALO_H * 128;
  static constexpr int PATCH_BYTES = (PATCH_DATA + 1023) / 1024 * 1024;
  static constexpr int PATCH_CHUNK = HALO_W * HALO_H * 16;
  static constexpr int STG_CHUNK = 128 * 128;
  static constexpr int PATCH_OFF = T2_BYTES;
  static constexpr int RING_OFF = PATCH_OFF + 2 * PATCH_BYTES;
  static constexpr int STG_OFF = RING_OFF + STAGES * SLOT;
  static constexpr int BAR_OFF = STG_OFF + 2 * STG_CHUNK;
  static constexpr int NUM_BARS = 2 * STAGES + 4 + 1;
  static constexpr int TOTAL = BAR_OFF + 8 * NUM_BARS + 1024;
};

template <int CM, bool RAGGED>
__global__ void __launch_bounds__(PERS_THREADS, 1)
conv_c23_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB2,
                const __grid_constant__ CUtensorMap tmB3, const __grid_constant__ CUtensorMap tmR,
                const __grid_constant__ CUtensorMap tmO, const ConvPersParams p, const float* __restrict__ scale2,
                const float* __restrict__ shift2) {
  using L = C23Smem<CM>;
  constexpr int NB2 = L::NB2, STAGES = L::STAGES;
  constexpr int KB = CM / 64;                      // 64-channel blocks of conv2's input and of conv3's K
  constexpr int N2C = CM / NB2, N3C = 4 * CM / 128;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* t2 = smem;
  uint8_t* patch = smem + L::PATCH_OFF;
  uint8_t* ring = smem + L::RING_OFF;
  uint8_t* stg = smem + L::STG_OFF;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::BAR_OFF);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* pfull_bar = empty_bar + STAGES;
  uint64_t* pempty_bar = pfull_bar + 2;
  uint64_t* res_bar = pempty_bar + 2;

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);
  const int lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB2);
    tma_prefetch_desc(&tmB3);
    tma_prefetch_desc(&tmR);
    tma_prefetch_desc(&tmO);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);
    }
    for (int s = 0; s < 2; ++s) {
      mbar_init(&pfull_bar[s], 1);
      mbar_init(&pempty_bar[s], 2);
    }
    mbar_init(res_bar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();

  if (warp < 4) {
    if (threadIdx.x == 0) {
      // ------------------------------------------------------------ producer
      uint32_t g = 0, gp = 0;
      auto load_w = [&](const CUtensorMap* m, int bytes, int k0, int n0) {
        const int s = g % STAGES;
        mbar_wait(&empty_bar[s], ((g / STAGES) & 1) ^ 1);
        mbar_expect_tx(&full_bar[s], bytes);
        tma_load_2d(ring + s * L::SLOT, m, &full_bar[s], k0, n0);
        ++g;
      };
      for (int t = blockIdx.x; t < p.total_tiles; t += gridDim.x) {
        const TileCoord c = decode_tile(p, t);
        for (int n2 = 0; n2 < N2C; ++n2)
          for (int kc = 0; kc < KB; ++kc, ++gp) {
            const int ps = gp % 2;
            mbar_wait(&pempty_bar[ps], ((gp / 2) & 1) ^ 1);
            mbar_expect_tx(&pfull_bar[ps], L::PATCH_DATA);
            tma_load_5d(patch + ps * L::PATCH_BYTES, &tmA, &pfull_bar[ps], 0, c.wo0 - 1, c.ho0 - 1, c.n0, kc * 8);
            for (int tap = 0; tap < 9; ++tap) load_w(&tmB2, NB2 * 128, (tap * KB + kc) * 64, n2 * NB2);
          }
        for (int n3 = 0; n3 < N3C; ++n3)
          for (int kc = 0; kc < KB; ++kc) load_w(&tmB3, 128 * 128, kc * 64, n3 * 128);
      }
    }
    return;
  }

  // ---------------------------------------------------------------- consumers
  const int wg = (warp >> 2) - 1;
  const int ctid = static_cast<int>(threadIdx.x) - 128;
  const bool leader = ctid == 0;
  const bool wg_leader = (ctid & 127) == 0;
  const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const int t4 = lane & 3;
  const uint32_t t2_addr = smem_u32(t2), stg_addr = smem_u32(stg);
  float acc[64];
#pragma unroll
  for (int j = 0; j < 64; ++j) acc[j] = 0.f;

  uint32_t g = 0, gp = 0, rc = 0;
  for (int t = blockIdx.x; t < p.total_tiles; t += gridDim.x) {
    const TileCoord c = decode_tile(p, t);

    // ------------------------------------------------------------ conv2 -> T2
    for (int n2 = 0; n2 < N2C; ++n2) {
      bool prev_last = false;
      for (int kc = 0; kc < KB; ++kc, ++gp) {
        const int ps = gp % 2;
        mbar_wait(&pfull_bar[ps], (gp / 2) & 1);
        const uint32_t pa = smem_u32(patch + ps * L::PATCH_BYTES);
        for (int tap = 0; tap < 9; ++tap, ++g) {
          const int s = g % STAGES;
          const int kh = tap / 3, kw = tap - 3 * (tap / 3);
          mbar_wait(&full_bar[s], (g / STAGES) & 1);
          const uint64_t adesc = gmma_desc_noswizzle(pa + ((wg * 8 + kh) * HALO_W + kw) * 16, L::PATCH_CHUNK, HALO_W * 16);
          const uint64_t bdesc = gmma_desc_sw128(smem_u32(ring + s * L::SLOT));
#pragma unroll
          for (int j = 0; j < 64; ++j) fence_operand(acc[j]);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < 4; ++k)
            wgmma_f16<NB2>(acc, adesc + ((2 * k * L::PATCH_CHUNK) >> 4), bdesc + 2 * k, (kc | tap | k) != 0);
          wgmma_commit();
          wgmma_wait<1>();
#pragma unroll
          for (int j = 0; j < 64; ++j) fence_operand(acc[j]);
          if ((kc | tap) != 0 && wg_leader) {
            mbar_arrive(&empty_bar[(g - 1) % STAGES]);
            if (prev_last) mbar_arrive(&pempty_bar[(gp - 1) % 2]);
          }
          prev_last = tap == 8;
        }
      }
      wgmma_wait<0>();
#pragma unroll
      for (int j = 0; j < 64; ++j) fence_operand(acc[j]);
      if (wg_leader) {
        mbar_arrive(&empty_bar[(g - 1) % STAGES]);
        mbar_arrive(&pempty_bar[(gp - 1) % 2]);
      }
      // BN + ReLU -> fp16 into T2 (the previous tile's conv3 MMAs of this warpgroup have completed: wait<0> above)
#pragma unroll
      for (int j = 0; j < NB2 / 8; ++j) {
        const int col = n2 * NB2 + j * 8 + 2 * t4;
        const float2 sc = __ldg(reinterpret_cast<const float2*>(scale2 + col));
        const float2 sh = __ldg(reinterpret_cast<const float2*>(shift2 + col));
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = r0 + 8 * h;
          const int jj = (n2 * NB2) / 8 + j;       // 16-byte unit index over all CM channels
          const uint32_t sp = t2_addr + (jj >> 3) * (128 * 128) + r * 128 + (((jj & 7) ^ (r & 7)) << 4) + t4 * 4;
          const float v0 = fmaxf(fmaf(acc[4 * j + 2 * h], sc.x, sh.x), 0.f);
          const float v1 = fmaxf(fmaf(acc[4 * j + 2 * h + 1], sc.y, sh.y), 0.f);
          asm volatile("st.shared.u32 [%0], %1;" ::"r"(sp), "r"(pack_h2(v0, v1)) : "memory");
        }
      }
    }
    fence_proxy_async_smem();                      // T2 (generic-proxy writes) -> visible to this warpgroup's wgmma
    named_bar_sync(2 + wg, 128);

    // ------------------------------------------------------------ conv3 (+ residual) -> out
    for (int n3 = 0; n3 < N3C; ++n3, ++rc) {
      if (leader) {
        bulk_wait_read<0>();                        // the previous chunk's stores have left the staging buffers
        mbar_expect_tx(res_bar, 2 * L::STG_CHUNK);
        for (int ch = 0; ch < 2; ++ch)
          tma_load_4d(stg + ch * L::STG_CHUNK, &tmR, res_bar, n3 * 128 + ch * 64, c.wo0, c.ho0, c.n0);
      }
      for (int kc = 0; kc < KB; ++kc, ++g) {
        const int s = g % STAGES;
        mbar_wait(&full_bar[s], (g / STAGES) & 1);
        const uint64_t adesc = gmma_desc_sw128(t2_addr + kc * (128 * 128) + wg * 64 * 128);
        const uint64_t bdesc = gmma_desc_sw128(smem_u32(ring + s * L::SLOT));
#pragma unroll
        for (int j = 0; j < 64; ++j) fence_operand(acc[j]);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_f16<128>(acc, adesc + 2 * k, bdesc + 2 * k, (kc | k) != 0);
        wgmma_commit();
        wgmma_wait<1>();
#pragma unroll
        for (int j = 0; j < 64; ++j) fence_operand(acc[j]);
        if (kc > 0 && wg_leader) mbar_arrive(&empty_bar[(g - 1) % STAGES]);
      }
      wgmma_wait<0>();
#pragma unroll
      for (int j = 0; j < 64; ++j) fence_operand(acc[j]);
      if (wg_leader) mbar_arrive(&empty_bar[(g - 1) % STAGES]);

      mbar_wait(res_bar, rc & 1);                   // residual chunk has landed in the staging buffers
      // ragged batch: conv2's T2 rows outside the image are not masked - they feed conv3 at the same pixel only, whose
      // output is zeroed here
      bool keep[2] = {true, true};
      if constexpr (RAGGED) {
        keep[0] = row_in_extent(p, c.m_tile, c.wo0, c.ho0, c.n0, r0);
        keep[1] = row_in_extent(p, c.m_tile, c.wo0, c.ho0, c.n0, r0 + 8);
      }
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int col = j * 8 + 2 * t4;
        const float2 sc = __ldg(reinterpret_cast<const float2*>(p.scale + n3 * 128 + col));
        const float2 sh = __ldg(reinterpret_cast<const float2*>(p.shift + n3 * 128 + col));
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = r0 + 8 * h;
          const uint32_t sp = stg_addr + (j >> 3) * L::STG_CHUNK + r * 128 + (((j & 7) ^ (r & 7)) << 4) + t4 * 4;
          float v0 = fmaf(acc[4 * j + 2 * h], sc.x, sh.x);
          float v1 = fmaf(acc[4 * j + 2 * h + 1], sc.y, sh.y);
          uint32_t rv;
          asm volatile("ld.shared.u32 %0, [%1];" : "=r"(rv) : "r"(sp));
          const float2 f = unpack_h2(rv);
          v0 = keep[h] ? fmaxf(v0 + f.x, 0.f) : 0.f;
          v1 = keep[h] ? fmaxf(v1 + f.y, 0.f) : 0.f;
          asm volatile("st.shared.u32 [%0], %1;" ::"r"(sp), "r"(pack_h2(v0, v1)) : "memory");
        }
      }
      fence_proxy_async_smem();
      named_bar_sync(1, PERS_CONSUMER_THREADS);
      if (leader) {
        for (int ch = 0; ch < 2; ++ch) tma_store_4d(&tmO, stg + ch * L::STG_CHUNK, n3 * 128 + ch * 64, c.wo0, c.ho0, c.n0);
        bulk_commit();
      }
    }
  }
  if (leader) bulk_wait<0>();
}

template <int CM, bool RAGGED = false>
int conv_c23_launch(const CUtensorMap& tmA, const CUtensorMap& tmB2, const CUtensorMap& tmB3, const CUtensorMap& tmR,
                    const CUtensorMap& tmO, const ConvPersParams& p, const float* scale2, const float* shift2, int num_sms,
                    cudaStream_t stream) {
  using L = C23Smem<CM>;
  static_assert(L::TOTAL <= 232448, "shared memory budget exceeded");
  auto kern = conv_c23_kernel<CM, RAGGED>;
  static std::atomic<uint64_t> attr_done{0};
  if (first_launch_on_device(attr_done))
    DIRB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L::TOTAL));
  const int grid = p.total_tiles < num_sms ? p.total_tiles : num_sms;
  DIRB_CUDA(launch_pdl(kern, dim3(grid), dim3(PERS_THREADS), L::TOTAL, stream, tmA, tmB2, tmB3, tmR, tmO, p, scale2, shift2));
  count_launch();
  return 0;
}

}  // namespace dirb
