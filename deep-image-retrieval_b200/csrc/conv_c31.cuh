// Two identity Bottlenecks b, b+1 joined in one persistent wgmma kernel for sm_90a: block b's conv3 (1x1, Cm -> 4 Cm)
// + BN + residual + ReLU and block b+1's conv1 (1x1, 4 Cm -> Cm) + BN + ReLU, per flat tile of 128 pixels
// (resnet.py:75-85).  Block b's output X is written once (it is block b+1's residual) and never read back for conv1.
//
//   weights         conv3's boxes (per chunk c of X: W3 rows N3 c .., K blocks 0 .. Cm/64 - 1), then conv1's (W1 K
//                   blocks of chunk c, each as Cm / NB1 boxes of NB1 rows) stream through one ring of 16 KB slots in the
//                   order the consumers read them; warpgroup 0's leader issues them (note 5)
//   warpgroups 0-1  consumers: warpgroup w owns pixel rows 64w .. 64w+63 of every tile and issues its own TMA traffic
//                   (leader thread): its T2 rows (resident, K-major, 128-byte swizzled), its residual rows, its X and T1
//                   stores.  Per chunk c it
//                     1. runs conv3 over K = Cm into acc3 (wgmma m64n128k16, N3 = 128 channels, K ascending, as the
//                        unfused +res launch),
//                     2. applies the conv_pers.cuh epilogue (BN, residual TMA-loaded into staging buffer c % NBUF,
//                        ReLU, ragged rows zeroed, fp16) into that staging buffer and TMA-stores it to X,
//                     3. runs conv1 over K = [N3 c, N3 c + N3) into acc1 (64 x Cm fp32, wgmma m64nNB1k16 per NB1
//                        output channels) with the staging buffer as A operand: the swizzled staging layout IS the
//                        K-major wgmma layout, so the chunk is used without a copy.
//                   After the last chunk acc1 gets BN + ReLU (ragged rows zeroed) and goes to T1 through the staging
//                   buffers.
// Each output element is accumulated in the K order of the unfused launches (a wgmma's result for one element does not
// depend on its N, which the unfused launches already vary with the batch) and with the same epilogue code, so X and
// T1 equal the two-kernel path bit for bit.  Ragged batches: conv1 reads the X rows the
// conv3 epilogue zeroed, exactly what the unfused conv1 reads from HBM.
//
// Protocol (g = ring slot counter, common to both consumer warpgroups; q = chunk counter of the CTA, i = tile
// counter of the CTA):
//   1. ring: one wgmma group per slot.  After committing group g a warpgroup waits for group g - 1 (wait_group 1) and
//      its leader releases that slot; before an epilogue, wait_group 0 and the last slot is released.  Each empty
//      barrier expects one arrival per consumer warpgroup.  Warpgroup 0's leader, after its own release of fill f,
//      waits for warpgroup 1's and loads fill f + STAGES into the slot: it only ever waits for a slot warpgroup 1 can
//      reach with fills already issued, so neither warpgroup can block the other for good.
//   2. staging buffer b = q % NBUF (per warpgroup: 64 rows x N3 channels): the residual of chunk q lands on
//      res_bar[w][b], phase (q / NBUF) & 1 (NBUF divides the chunks per tile).  It is loaded after chunk q - 1's
//      epilogue, once all but the latest bulk group have read smem (the buffer's last readers: the store of chunk
//      q - NBUF and conv1 of that chunk, which wait_group 0 before a later epilogue finished) - except chunk 0 of a tile,
//      which waits for the previous tile's T1 store (it used every buffer) to have read everything.
//   3. T2 rows of tile i land on t2_bar[w], phase i & 1; the next tile's rows are loaded after the last chunk's epilogue
//      (conv3 done in all four warps: wait_group 0, then the epilogue's named barrier).
//   4. staging writes (generic proxy) reach the TMA stores and conv1's wgmma through fence.proxy.async + the warpgroup's
//      named barrier 1 + w; T1's staging writes wait for every store of the tile to have read the buffers.
//   5. registers: acc1 (Cm / 2) + acc3 (N3 / 2) per consumer thread, 192 at Cm = 256.  With a producer warpgroup the
//      launch gives 168 per thread and setmaxnreg.inc 232 lets the consumers' code use more - but ptxas does so only
//      for code without a trap, and mbar_wait's spin limit traps: built that way this kernel spilled 2 KB per thread at
//      Cm = 256 (1 KB with 64-channel conv3 chunks), while a trap-free toy with 200 live values did not spill.  With
//      the two consumer warpgroups alone every thread gets 255 and no instantiation spills.  The cost: warpgroup 0's
//      leader refills a slot only after warpgroup 1's release, so the warpgroups stay within about one slot of each
//      other and one's epilogue does not run under the other's MMAs.
//   The protocol is modelled in tests/c31_model.py (tests/test_c31_protocol.py).
#pragma once
#include "conv_pers.cuh"

namespace dirb {

template <int CM>
struct C31Smem {
  static constexpr int NB1 = CM < 128 ? CM : 128;                    // conv1 output channels per wgmma
  static constexpr int N3 = 128;                                     // conv3 output channels per chunk
  static constexpr int NBUF = 256 / N3;                              // staging buffers of N3 channels
  static constexpr int CHUNK = 128 * 128;                            // 128 rows x 64 channels fp16, 128-byte swizzled
  static constexpr int SLOT = 128 * 128;                             // weight box, up to 128 rows x 64 K
  static constexpr int T2_BYTES = (CM / 64) * CHUNK;
  static constexpr int STG_OFF = T2_BYTES;
  static constexpr int STG_BYTES = 4 * CHUNK;                        // 256 channels: T1 (up to Cm) or NBUF X chunks
  static constexpr int RING_OFF = STG_OFF + STG_BYTES;
  static constexpr int NUM_BARS_MAX = 2 * 8 + 2 + 8;
  static constexpr int RING_BUDGET = 232448 - 1024 - 8 * NUM_BARS_MAX - RING_OFF;
  static constexpr int STAGES = RING_BUDGET / SLOT < 8 ? RING_BUDGET / SLOT : 8;
  static constexpr int BAR_OFF = RING_OFF + STAGES * SLOT;
  static constexpr int NUM_BARS = 2 * STAGES + 2 + 2 * NBUF;         // ring full / empty, T2 and residual per warpgroup
  static constexpr int TOTAL = BAR_OFF + 8 * NUM_BARS + 1024;        // + alignment slack
};

// One ring slot = one wgmma group: acc (+)= A (64 x 64, descriptor adesc) * slot^T (N x 64); then the previous group is
// complete and release(g - 1) hands its slot back (protocol 1).
template <int N, int STAGES, class Release>
__device__ __forceinline__ void c31_mma_slot(float (&acc)[N / 2], uint64_t adesc, bool accumulate, const uint8_t* ring,
                                             uint64_t* full_bar, uint32_t& g, bool& held, const Release& release) {
  const int s = g % STAGES;
  mbar_wait(&full_bar[s], (g / STAGES) & 1);
  const uint64_t bdesc = gmma_desc_sw128(smem_u32(ring + s * (128 * 128)));   // C31Smem::SLOT
#pragma unroll
  for (int j = 0; j < N / 2; ++j) fence_operand(acc[j]);
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < 4; ++k) wgmma_f16<N>(acc, adesc + 2 * k, bdesc + 2 * k, accumulate || k != 0);
  wgmma_commit();
  wgmma_wait<1>();
#pragma unroll
  for (int j = 0; j < N / 2; ++j) fence_operand(acc[j]);
  if (held) release(g - 1);
  held = true;
  ++g;
}

constexpr int C31_THREADS = 256;   // two consumer warpgroups, no producer warp (note 5)

template <int CM, bool RAGGED>
__global__ void __launch_bounds__(C31_THREADS, 1)
conv_c31_kernel(const __grid_constant__ CUtensorMap tmT2, const __grid_constant__ CUtensorMap tmW3,
                const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmY,
                const __grid_constant__ CUtensorMap tmW1, const __grid_constant__ CUtensorMap tmT1, const ConvPersParams p,
                const float* __restrict__ scale1, const float* __restrict__ shift1) {
  using L = C31Smem<CM>;
  constexpr int STAGES = L::STAGES, NB1 = L::NB1, N3 = L::N3, NBUF = L::NBUF, CHUNK = L::CHUNK;
  constexpr int KB = CM / 64;                      // 64-channel blocks of T2 (conv3's K) and of T1
  constexpr int NC = 4 * CM / N3;                  // chunks of X
  constexpr int NH1 = CM / NB1;                    // conv1 wgmmas per K step
  constexpr int NS = N3 / 64;                      // 64-channel blocks per chunk (staging chunks, conv1 K steps)
  static_assert(NC % NBUF == 0, "every tile starts at staging buffer 0 (protocol 2)");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* t2 = smem;
  uint8_t* stg = smem + L::STG_OFF;
  uint8_t* ring = smem + L::RING_OFF;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::BAR_OFF);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* t2_bar = empty_bar + STAGES;           // [2]
  uint64_t* res_bar = t2_bar + 2;                  // [2][NBUF]

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);
  const int lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmT2);
    tma_prefetch_desc(&tmW3);
    tma_prefetch_desc(&tmX);
    tma_prefetch_desc(&tmY);
    tma_prefetch_desc(&tmW1);
    tma_prefetch_desc(&tmT1);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);
    }
    for (int b = 0; b < 2 + 2 * NBUF; ++b) mbar_init(&t2_bar[b], 1);   // t2_bar[2], res_bar[2][NBUF]
    fence_mbar_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();

  // ---------------------------------------------------------------- consumers
  const int wg = warp >> 2;
  const bool wg_leader = (threadIdx.x & 127) == 0;
  const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // this thread's rows of the tile: r0, r0 + 8
  const int t4 = lane & 3;
  const int half = wg * 64 * 128;                  // this warpgroup's rows inside a 128-row chunk
  const uint32_t t2_addr = smem_u32(t2), stg_addr = smem_u32(stg);
  uint64_t* t2_w = t2_bar + wg;
  uint64_t* res_w = res_bar + NBUF * wg;
  const int bar = 1 + wg;

  // ring fill f: the weight boxes of one tile (NC chunks of KB W3 boxes, then NS x NH1 W1 boxes) repeat for every tile
  // of the CTA.  Warpgroup 0's leader refills a slot as soon as both warpgroups have released it.
  constexpr uint32_t PER_CHUNK = KB + NS * NH1;
  const uint32_t n_fills = static_cast<uint32_t>((p.total_tiles - static_cast<int>(blockIdx.x) + static_cast<int>(gridDim.x) - 1) /
                                                 static_cast<int>(gridDim.x)) * NC * PER_CHUNK;
  auto fill = [&](uint32_t f) {
    if (f >= n_fills) return;
    const int s = f % STAGES;
    mbar_wait(&empty_bar[s], ((f / STAGES) & 1) ^ 1);
    const int c = (f / PER_CHUNK) % NC;
    int e = f % PER_CHUNK;
    if (e < KB) {
      mbar_expect_tx(&full_bar[s], N3 * 128);
      tma_load_2d(ring + s * L::SLOT, &tmW3, &full_bar[s], e * 64, c * N3);
    } else {
      e -= KB;
      mbar_expect_tx(&full_bar[s], NB1 * 128);
      tma_load_2d(ring + s * L::SLOT, &tmW1, &full_bar[s], c * N3 + (e / NH1) * 64, (e % NH1) * NB1);
    }
  };
  auto release = [&](uint32_t f) {
    if (wg_leader) {
      mbar_arrive(&empty_bar[f % STAGES]);
      if (wg == 0) fill(f + STAGES);
    }
  };
  if (wg == 0 && wg_leader)
    for (int f = 0; f < STAGES; ++f) fill(f);

  auto load_t2 = [&](int t) {
    mbar_expect_tx(t2_w, KB * CHUNK / 2);
    for (int kc = 0; kc < KB; ++kc) tma_load_2d(t2 + kc * CHUNK + half, &tmT2, t2_w, kc * 64, t * 128 + wg * 64);
  };
  auto load_res = [&](int t, int c) {
    const int b = c % NBUF;
    mbar_expect_tx(&res_w[b], NS * CHUNK / 2);
    for (int h = 0; h < NS; ++h)
      tma_load_2d(stg + (NS * b + h) * CHUNK + half, &tmX, &res_w[b], c * N3 + h * 64, t * 128 + wg * 64);
  };

  float acc3[1][N3 / 2];
  float acc1[NH1][1][NB1 / 2];
  uint32_t g = 0, q = 0;
  bool held = false;                               // slot g - 1 has not been released yet
  if (wg_leader && static_cast<int>(blockIdx.x) < p.total_tiles) {
    load_t2(blockIdx.x);
    load_res(blockIdx.x, 0);
  }
  for (int t = blockIdx.x, i = 0; t < p.total_tiles; t += gridDim.x, ++i) {
    const int next = t + static_cast<int>(gridDim.x);
    uint32_t keep = 3;
    if constexpr (RAGGED) {
      keep = row_in_extent(p, t, 0, 0, 0, r0) ? 1u : 0u;
      keep |= row_in_extent(p, t, 0, 0, 0, r0 + 8) ? 2u : 0u;
    }
    mbar_wait(t2_w, i & 1);
    for (int c = 0; c < NC; ++c, ++q) {
      const int b = c % NBUF;
      // ---------------------------------------------------------- conv3 chunk c
      for (int kc = 0; kc < KB; ++kc)
        c31_mma_slot<N3, STAGES>(acc3[0], gmma_desc_sw128(t2_addr + kc * CHUNK + half), kc != 0, ring, full_bar, g, held,
                                 release);
      wgmma_wait<0>();
#pragma unroll
      for (int j = 0; j < N3 / 2; ++j) fence_operand(acc3[0][j]);
      release(g - 1);
      held = false;
      // ---------------------------------------------------------- + BN + residual + ReLU -> X (staging buffer b)
      mbar_wait(&res_w[b], (q / NBUF) & 1);
      conv_epilogue_to_staging<N3, 1, RAGGED>(acc3, stg_addr + NS * b * CHUNK, r0, t4, p.scale + c * N3,
                                              p.shift + c * N3, true, true, keep);
      fence_proxy_async_smem();
      named_bar_sync(bar, 128);
      if (wg_leader) {
        for (int h = 0; h < NS; ++h) tma_store_2d(&tmY, stg + (NS * b + h) * CHUNK + half, c * N3 + h * 64, t * 128 + wg * 64);
        bulk_commit();
        if (c + 1 < NC) {
          bulk_wait_read<1>();
          load_res(t, c + 1);
        } else if (next < p.total_tiles) {
          load_t2(next);
        }
      }
      // ---------------------------------------------------------- conv1 of block b+1, K = [N3 c, N3 c + N3)
#pragma unroll
      for (int kk = 0; kk < NS; ++kk)
#pragma unroll
        for (int nh = 0; nh < NH1; ++nh)
          c31_mma_slot<NB1, STAGES>(acc1[nh][0], gmma_desc_sw128(stg_addr + (NS * b + kk) * CHUNK + half), (c | kk) != 0,
                                    ring, full_bar, g, held, release);
    }
    wgmma_wait<0>();
#pragma unroll
    for (int nh = 0; nh < NH1; ++nh)
#pragma unroll
      for (int j = 0; j < NB1 / 2; ++j) fence_operand(acc1[nh][0][j]);
    release(g - 1);
    held = false;
    // ------------------------------------------------------------ + BN + ReLU -> T1 (both staging buffers)
    if (wg_leader) bulk_wait_read<0>();
    named_bar_sync(bar, 128);
#pragma unroll
    for (int nh = 0; nh < NH1; ++nh)
      conv_epilogue_to_staging<NB1, 1, RAGGED>(acc1[nh], stg_addr + nh * (NB1 / 64) * CHUNK, r0, t4, scale1 + nh * NB1,
                                               shift1 + nh * NB1, false, true, keep);
    fence_proxy_async_smem();
    named_bar_sync(bar, 128);
    if (wg_leader) {
      for (int kc = 0; kc < KB; ++kc) tma_store_2d(&tmT1, stg + kc * CHUNK + half, kc * 64, t * 128 + wg * 64);
      bulk_commit();
      if (next < p.total_tiles) {
        bulk_wait_read<0>();
        load_res(next, 0);
      }
    }
  }
  if (wg_leader) bulk_wait<0>();                   // all output bytes written before the CTA retires
}

template <int CM, bool RAGGED = false>
int conv_c31_launch(const CUtensorMap& tmT2, const CUtensorMap& tmW3, const CUtensorMap& tmX, const CUtensorMap& tmY,
                    const CUtensorMap& tmW1, const CUtensorMap& tmT1, const ConvPersParams& p, const float* scale1,
                    const float* shift1, int num_sms, cudaStream_t stream) {
  using L = C31Smem<CM>;
  static_assert(L::TOTAL <= 232448, "shared memory budget exceeded");
  auto kern = conv_c31_kernel<CM, RAGGED>;
  static std::atomic<uint64_t> attr_done{0};
  if (first_launch_on_device(attr_done))
    DIRB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L::TOTAL));
  const int grid = p.total_tiles < num_sms ? p.total_tiles : num_sms;
  DIRB_CUDA(launch_pdl(kern, dim3(grid), dim3(C31_THREADS), L::TOTAL, stream, tmT2, tmW3, tmX, tmY, tmW1, tmT1, p, scale1,
                       shift1));
  count_launch();
  return 0;
}

}  // namespace dirb
