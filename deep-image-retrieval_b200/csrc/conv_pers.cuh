// Persistent wgmma implicit-GEMM convolution + BN + residual + ReLU for sm_90a, also the similarity / whitening GEMM.
//
// One CTA per SM loops over output tiles (128 pixels x BN channels, BN = 64 or 128); three warpgroups:
//
//   warpgroup 0     TMA producer (one thread): A (128x64 activation patch) and B (BNx64 weights) into a STAGES-deep
//                   shared-memory ring; it runs ahead across tiles, so the next tile's operands stream in while the
//                   consumers run the epilogue of the current one
//   warpgroups 1-2  consumers: warpgroup 1 + w owns accumulator rows 64w .. 64w+63 of the tile (wgmma m64nBNk16, fp32
//                   accumulators in registers, 4 x K=16 per ring slot).  The convolution epilogue applies BN
//                   scale/shift (+ residual) (+ ReLU) -> fp16 into 128-byte-swizzled staging buffers (one per 64
//                   channels) and one thread TMA-stores them (the store clips ragged edges by itself).  The residual tile
//                   is TMA-loaded into the same staging buffers when the tile starts, so it lands during the main loop.
//                   When every CTA gets three tiles or more, the convolution epilogue runs in ping-pong mode instead: each
//                   consumer warpgroup takes whole tiles, alternately, and its epilogue overlaps the other's MMAs (PP).
//
// HALO mode (3x3 / stride 1 / pad 1, 8 x 16 output pixels per tile): per 64-channel block ONE 5-D TMA box brings the
// 10 x 18 input patch (zero padding from out-of-bounds fill) into a patch ring, channel-chunk-major without swizzle, and
// the nine taps are nine wgmma descriptors with shifted start addresses into it; the operand ring holds weight tiles
// only.  The patch crosses the L2 -> SM path once instead of nine times.
//
// A operand addressing: flat rows [M][K] (2-D tensor map) or an NHWC activation read as an implicit-GEMM operand: for
// filter tap (kh,kw) and channel block kc the 128 rows of the tile are a (nb x th x tw) patch of output pixels, fetched
// by ONE 4-D TMA box at input offset (stride*ho0+kh-pad, stride*wo0+kw-pad); padding and ragged edges come from TMA
// out-of-bounds zero fill, stride-2 convolutions from the tensor map's element stride.
#pragma once
#include "common.h"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace dirb {

enum { PERS_EPI_CONV = 0, PERS_EPI_SIM_DENSE = 1, PERS_EPI_SIM_FILTER = 2, PERS_EPI_SIM_GMAX = 3, PERS_EPI_F32 = 4,
       PERS_EPI_SIM_JOIN = 5, PERS_EPI_SIM_LGMAX = 6, PERS_EPI_SIM_LFILTER = 7, PERS_EPI_SIM_FILTER_ALLOW = 8 };

struct ConvPersParams {
  int a_spatial, taps, kw_taps, cin_blocks, stride, pad;
  int tw, th, nb, tiles_w, tiles_h;
  int n_tiles, total_tiles;
  int m_fastest, m_tiles;      // tile order: 0 = n-tile fastest (convolutions: CTAs share the activation tile),
                               // 1 = m-tile fastest (search: CTAs running together share the streamed database tile)
  int has_res, relu;
  // fused projection shortcut (block 0 of a layer): k-iterations >= k_split read their A tile from a SECOND
  // activation tensor (tensor map tmR, spatial boxes with element stride a2_stride baked into the map) - the
  // block input x of the 1x1 downsample conv - while the weights are the K-concatenation [W3*s3 | Wd*sd].
  int k_split, a2_stride;
  // PERS_EPI_F32 (whitening): fp32-accurate product from fp16 hi/lo splits, K = 3 parts of k_per_part blocks:
  // (A_hi, B_lo), (A_lo, B_hi), (A_hi, B_hi) with A_lo in tensor map tmR and B_lo in tmO; epilogue = column scale,
  // fp32 store to dense[M][dense_ld].
  int k_per_part;
  const float* scale;
  const float* shift;
  // similarity epilogues (search.cu): D[q][n] = <query q, database row n>
  int M, N;                    // valid queries / database rows of this launch
  float* dense;                // [M][dense_ld] fp32 scores                     (PERS_EPI_SIM_DENSE)
  int64_t dense_ld;
  const float* thr;            // [M] per-query threshold                       (PERS_EPI_SIM_FILTER / _JOIN)
  unsigned long long* cand;    // [M][cand_cap] packed (score bits << 32 | row)
  int* cand_cnt;               // [M]
  int cand_cap;
  // Device-side launch predicate (retry passes of the search): when non-null the whole grid returns at once unless
  // *gate != 0.  The value was written by the previous kernel of the stream, so it is read after pdl_wait().
  const int* gate;
  // Ragged batches (convolution epilogue): image n of the output tensor holds a picture of ext[n*ext_ld] x
  // ext[n*ext_ld + 1] pixels in its top-left corner; every output pixel outside it is written as 0.  ext_n = images in
  // the tensor, out_h / out_w = its spatial dims (the flat 2-D mode decodes a row index with them).  kc_major (spatial
  // tiles with nb == 1 only): kc_major[n*ext_ld] != 0 walks image n's K loop channel block outer, tap inner - the
  // order of the HALO mode - so its bits equal those of a HALO launch.  Null = a plain dense batch.
  const int* ext;
  const int* kc_major;
  int ext_ld, ext_n, out_h, out_w;
  // list epilogues (PERS_EPI_SIM_LGMAX / _LFILTER, the inverted-file search): tile t is entry t of a device-built table
  // {A row, B row, column tile of the list, valid rows | valid columns << 16}.  A row s of the packed queries belongs to
  // query slot_q[s]; B row b of the list-ordered database is database row perm[b].  LGMAX writes the maximum of group g
  // of A row s's list to dense[gbase[s] + g]; LFILTER appends (score, perm[b]) to query slot_q[s]'s candidate list.
  const int4* tiles;
  const int* slot_q;
  const int64_t* perm;
  const int64_t* gbase;
  // PERS_EPI_SIM_FILTER_ALLOW (filtered search): the filter pass keeps column n of query row q only if bit allow_bit0 + n
  // of the allow bitmap's row q is set (word b >> 5, bit b & 31); allow_ld = words per query row, 0 = one row shared.
  const uint32_t* allow;
  int64_t allow_ld, allow_bit0;
};

// Whether accumulator row r of tile c lies inside its image's extent (ragged batches; true without an extent table).
__device__ __forceinline__ bool row_in_extent(const ConvPersParams& p, int m_tile, int wo0, int ho0, int n0, int r) {
  if (p.ext == nullptr) return true;
  int n, y, x;
  if (p.a_spatial) {
    x = wo0 + r % p.tw;
    y = ho0 + (r / p.tw) % p.th;
    n = n0 + r / (p.tw * p.th);
  } else {
    const int64_t m = static_cast<int64_t>(m_tile) * 128 + r;
    x = static_cast<int>(m % p.out_w);
    y = static_cast<int>((m / p.out_w) % p.out_h);
    n = static_cast<int>(m / (static_cast<int64_t>(p.out_w) * p.out_h));
  }
  if (n >= p.ext_n) return false;                  // beyond the tensor: the TMA store clips the row anyway
  return y < __ldg(p.ext + static_cast<int64_t>(n) * p.ext_ld) && x < __ldg(p.ext + static_cast<int64_t>(n) * p.ext_ld + 1);
}

// Convolution epilogue of one thread's accumulators (layout of wgmma.cuh): BN scale / shift (+ the residual already in
// the staging buffer) (+ ReLU), ragged rows zeroed (keep bit 2 * hf + h = row r0 + 64 * hf + 8 * h lies inside its
// image), fp16 into the staging buffer at stg_base: 128 rows x 64 channels per 128-byte-swizzled chunk, one chunk per 64
// of the BN columns.  scale / shift point at the first column.
template <int BN, int NH, bool RAGGED>
__device__ __forceinline__ void conv_epilogue_to_staging(const float (&acc)[NH][BN / 2], uint32_t stg_base, int r0, int t4,
                                                         const float* scale, const float* shift, bool has_res, bool relu,
                                                         uint32_t keep) {
  constexpr int STG_CHUNK = 128 * 128;
  // this thread's rows r0 + 64 * hf + 8 * h all share r0 & 7, so their 128-byte swizzle (16-byte unit j ^ (r & 7)) is
  // the same and the rows differ by immediate offsets
  const uint32_t stg_addr = stg_base + r0 * 128 + t4 * 4;
  const int rsw = r0 & 7;
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int col = j * 8 + 2 * t4;
    const float2 sc = __ldg(reinterpret_cast<const float2*>(scale + col));
    const float2 sh = __ldg(reinterpret_cast<const float2*>(shift + col));
#pragma unroll
    for (int hf = 0; hf < NH; ++hf) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint32_t sp = stg_addr + (j >> 3) * STG_CHUNK + (64 * hf + 8 * h) * 128 + (((j & 7) ^ rsw) << 4);
        float v0 = fmaf(acc[hf][4 * j + 2 * h], sc.x, sh.x);
        float v1 = fmaf(acc[hf][4 * j + 2 * h + 1], sc.y, sh.y);
        if (has_res) {
          uint32_t rv;
          asm volatile("ld.shared.u32 %0, [%1];" : "=r"(rv) : "r"(sp));
          const float2 f = unpack_h2(rv);
          v0 += f.x;
          v1 += f.y;
        }
        if (relu) {
          v0 = fmaxf(v0, 0.f);
          v1 = fmaxf(v1, 0.f);
        }
        if (RAGGED && !((keep >> (2 * hf + h)) & 1)) {                     // ragged batch: outside the image = zero padding of the next layer
          v0 = 0.f;
          v1 = 0.f;
        }
        asm volatile("st.shared.u32 [%0], %1;" ::"r"(sp), "r"(pack_h2(v0, v1)) : "memory");
      }
    }
  }
}

// HALO (3x3 / stride 1 / pad 1, 8 x 16 output tiles): the ring holds weight tiles only; per 64-channel block ONE TMA box
// brings the 10 x 18 input patch into a separate ring of NP patch slots, and the nine taps read it as shifted views.
// PP (ping-pong consumers, convolution epilogue only): each consumer warpgroup has its own staging buffers, residual
// barrier and mainloop-handover barrier.
template <int BN, int STAGES, int EPI = 0, bool HALO = false, bool PP = false>
struct ConvPersSmem {
  static constexpr int A_BYTES = HALO ? 0 : 128 * 128;
  static constexpr int B_BYTES = BN * 128;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int NP = HALO ? 2 : 0;                            // patch slots
  static constexpr int PATCH_DATA = HALO_W * HALO_H * 128;           // 64 channels of HALO_W x HALO_H pixels
  static constexpr int PATCH_BYTES = (PATCH_DATA + 1023) / 1024 * 1024;
  static constexpr int PATCH_CHUNK = HALO_W * HALO_H * 16;           // one 8-channel chunk of the patch
  static constexpr int PATCH_OFF = STAGES * STAGE_BYTES;
  static constexpr int STG_CHUNK = 128 * 128;                        // 128 rows x 64 channels fp16
  static constexpr int STG_OFF = PATCH_OFF + NP * PATCH_BYTES;
  static constexpr int NWG_STG = PP ? 2 : 1;                         // staging sets: one per warpgroup in ping-pong
  static constexpr int WG_STG_BYTES = (EPI == 0) ? (BN / 64) * STG_CHUNK : 0;  // staging exists only for the conv epilogue
  static constexpr int STG_BYTES = NWG_STG * WG_STG_BYTES;
  static constexpr int BAR_OFF = STG_OFF + STG_BYTES;
  // ring full / empty, patch full / empty, residual (per staging set), ping-pong mainloop handover (2)
  static constexpr int NUM_BARS = 2 * STAGES + 2 * NP + NWG_STG + (PP ? 2 : 0);
  static constexpr int TOTAL = BAR_OFF + 8 * NUM_BARS + 1024;        // + alignment slack
};

constexpr int PERS_THREADS = 384;            // producer warpgroup + two consumer warpgroups
constexpr int PERS_CONSUMER_THREADS = 256;

struct TileCoord {
  int m_tile, n_tile, wo0, ho0, n0;
  int a_row, b_row, m_valid, n_valid;   // list tiles only (decode_tile_list)
};
__device__ __forceinline__ TileCoord decode_tile(const ConvPersParams& p, int t) {
  TileCoord c;
  if (p.m_fastest) {
    c.m_tile = t % p.m_tiles;
    c.n_tile = t / p.m_tiles;
  } else {
    c.n_tile = t % p.n_tiles;
    c.m_tile = t / p.n_tiles;
  }
  c.wo0 = c.ho0 = c.n0 = 0;
  if (p.a_spatial) {
    const int tx = c.m_tile % p.tiles_w;
    const int ty = (c.m_tile / p.tiles_w) % p.tiles_h;
    const int tb = c.m_tile / (p.tiles_w * p.tiles_h);
    c.wo0 = tx * p.tw;
    c.ho0 = ty * p.th;
    c.n0 = tb * p.nb;
  }
  return c;
}

// PERS_EPI_SIM_JOIN (self-join of a row block against itself and the rows after it): A rows and B rows start at the
// same database row, a multiple of 128, so tile (m, n) with n < m lies wholly below the diagonal and is never launched.
// The m_tiles x n_tiles grid (n_tiles >= m_tiles) keeps the tiles with n >= m, m fastest: column n < m_tiles holds
// n + 1 tiles, every later column m_tiles, so the launch has T_m (T_m + 1) / 2 + (T_n - T_m) T_m tiles.
__device__ __forceinline__ TileCoord decode_tile_tri(const ConvPersParams& p, int t) {
  TileCoord c;
  const int64_t mt = p.m_tiles;
  const int64_t tri = mt * (mt + 1) / 2;
  if (t < tri) {
    int64_t n = static_cast<int64_t>((sqrt(8.0 * t + 1.0) - 1.0) * 0.5);
    while (n * (n + 1) / 2 > t) --n;
    while ((n + 1) * (n + 2) / 2 <= t) ++n;
    c.n_tile = static_cast<int>(n);
    c.m_tile = static_cast<int>(t - n * (n + 1) / 2);
  } else {
    const int64_t u = t - tri;
    c.n_tile = static_cast<int>(mt + u / mt);
    c.m_tile = static_cast<int>(u % mt);
  }
  c.wo0 = c.ho0 = c.n0 = 0;
  return c;
}

// PERS_EPI_SIM_LGMAX / _LFILTER: one table entry per tile; a tile never spans two lists (n_tile = its column tile within
// the list), rows past m_valid are the zero padding of the list's query segment, columns past n_valid belong to the next
// list or lie past the last row.
template <int EPI>
constexpr bool pers_list_epi() { return EPI == PERS_EPI_SIM_LGMAX || EPI == PERS_EPI_SIM_LFILTER; }
__device__ __forceinline__ TileCoord decode_tile_list(const ConvPersParams& p, int t) {
  TileCoord c;
  const int4 e = __ldg(p.tiles + t);
  c.a_row = e.x;
  c.b_row = e.y;
  c.m_tile = 0;
  c.n_tile = e.z;
  c.m_valid = e.w & 0xffff;
  c.n_valid = e.w >> 16;
  c.wo0 = c.ho0 = c.n0 = 0;
  return c;
}

template <int EPI>
__device__ __forceinline__ TileCoord decode_any_tile(const ConvPersParams& p, int t) {
  if constexpr (EPI == PERS_EPI_SIM_JOIN) return decode_tile_tri(p, t);
  else if constexpr (pers_list_epi<EPI>()) return decode_tile_list(p, t);
  else return decode_tile(p, t);
}

// Writes one accumulator pair (two adjacent columns of one row) of the similarity / whitening epilogues.
__device__ __forceinline__ void store_dense_pair(const ConvPersParams& p, int64_t qi, int col, float v0, float v1) {
  float* dp = p.dense + qi * p.dense_ld + col;
  if (col + 1 < p.N && ((p.dense_ld & 1) == 0)) {
    *reinterpret_cast<float2*>(dp) = make_float2(v0, v1);
  } else {
    if (col < p.N) dp[0] = v0;
    if (col + 1 < p.N) dp[1] = v1;
  }
}

// RAGGED: the launch carries an extent table (ConvPersParams::ext); dense launches compile without its code.
//
// PP selects the consumer mode of the convolution epilogue:
//   false (cooperative)  both consumer warpgroups work on every tile, warpgroup w on rows 64w .. 64w+63; the tensor cores
//                        idle while the two run the epilogue together.
//   true  (ping-pong)    warpgroup w takes every other CTA-local tile (tile i -> warpgroup i & 1) and holds the whole
//                        128 x BN tile as acc[2][BN/2]; half h issues exactly the wgmmas that warpgroup h issues in the
//                        cooperative mode and runs its epilogue for rows 64h .. 64h+63, so the output is bit-identical.
//                        One warpgroup's epilogue runs under the other's main loop.
// Invariants of the ping-pong mode (tests/pingpong_model.py checks them on a model of the barriers):
//   1. ring parity: the main loops are handed over in tile order through mma_done[2] - only one warpgroup waits on the
//      operand / patch rings at a time, so no waiter is ever two phases ahead of a slot's barrier (try_wait.parity would
//      pass on the stale phase and the MMAs would read the wrong operands, with no hang and no trap).  Every consumer
//      WARP arrives (count 4, lane 0 after the warp's last full-barrier wait of the tile): wgmma synchronises a warp,
//      not a warpgroup, so one leader's arrival would not prove that its sibling warps have passed their own mma_done
//      wait - with k_iters == 1 a sibling could lag while the partner completes the barrier twice, and then wait on a
//      parity that never comes back;
//   2. slot counters at CTA-local tile i: g = i * k_iters (HALO: g = i * 9 * cin_blocks, gp = i * cin_blocks) - every
//      tile of a launch has the same number of k-iterations, kc_major only reorders them;
//   3. the ring-empty and patch-empty barriers expect one arrival per fill (template constant, not a launch parameter);
//   4. each warpgroup owns its staging buffers, residual barrier, bulk-store groups and 128-thread named barrier;
//   5. a warpgroup may get one tile fewer: its partner's last mma_done arrival then has no waiter, which an mbarrier
//      allows;
//   6. setmaxnreg moves registers from the producer warpgroup (40) to the consumers (232): 128 x 40 + 256 x 232 <= 64 K.
template <int BN, int STAGES, int EPI, bool HALO, bool RAGGED, bool PP>
__global__ void __launch_bounds__(PERS_THREADS, 1)
conv_pers_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const __grid_constant__ CUtensorMap tmR, const __grid_constant__ CUtensorMap tmO,
                 const ConvPersParams p) {
  using L = ConvPersSmem<BN, STAGES, EPI, HALO, PP>;
  constexpr int CHUNKS = BN / 64;
  constexpr int NH = PP ? 2 : 1;                    // 64-row accumulator halves per consumer warpgroup
  constexpr uint32_t EMPTY_ARRIVALS = PP ? 1 : 2;   // consumer warpgroups that read each fill (invariant 3)
  constexpr uint32_t MMA_DONE_ARRIVALS = 4;         // one per warp of the handing-over warpgroup (invariant 1)
  static_assert(!HALO || EPI == PERS_EPI_CONV, "the halo mode is a convolution");
  static_assert(!PP || EPI == PERS_EPI_CONV, "the ping-pong mode is a convolution epilogue");
  static_assert(!PP || 128 * 40 + 256 * 232 <= 65536, "register file exceeded");
  if (EPI != PERS_EPI_CONV && p.gate != nullptr) {   // uniform over the grid: nothing has been set up yet
    pdl_wait();
    if (*reinterpret_cast<const volatile int*>(p.gate) == 0) return;
  }
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* stg = smem + L::STG_OFF;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + L::BAR_OFF);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* pfull_bar = empty_bar + STAGES;
  uint64_t* pempty_bar = pfull_bar + L::NP;
  uint64_t* res_bar = pempty_bar + L::NP;           // [NWG_STG]
  uint64_t* mma_done = res_bar + L::NWG_STG;        // [2], ping-pong only
  uint8_t* patch = smem + L::PATCH_OFF;

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);
  const int lane = threadIdx.x & 31;
  const int k_iters = p.taps * p.cin_blocks;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if (EPI == PERS_EPI_CONV) tma_prefetch_desc(&tmO);
    if (EPI == PERS_EPI_CONV && (p.has_res || p.k_split > 0)) tma_prefetch_desc(&tmR);
    if (EPI == PERS_EPI_F32) { tma_prefetch_desc(&tmR); tma_prefetch_desc(&tmO); }
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], EMPTY_ARRIVALS);  // one arrival per consumer warpgroup reading the fill
    }
    for (int s = 0; s < L::NP; ++s) {
      mbar_init(&pfull_bar[s], 1);
      mbar_init(&pempty_bar[s], EMPTY_ARRIVALS);
    }
    for (int w = 0; w < L::NWG_STG; ++w) mbar_init(&res_bar[w], 1);
    if constexpr (PP) {
      mbar_init(&mma_done[0], MMA_DONE_ARRIVALS);
      mbar_init(&mma_done[1], MMA_DONE_ARRIVALS);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_launch_dependents();   // the next kernel may start its own prologue while this one runs / drains
  pdl_wait();                // everything below reads tensors written by the previous kernel of the stream

  if (warp < 4) {
    if constexpr (PP) setmaxnreg_dec<40>();        // all four producer warps, including the three that return at once
    if (threadIdx.x == 0) {
      // ------------------------------------------------------------ A/B producer
      uint32_t g = 0;  // ring slot counter, runs across tiles
      uint32_t gp = 0;  // patch slot counter (HALO)
      for (int t = blockIdx.x; t < p.total_tiles; t += gridDim.x) {
        const TileCoord c = decode_any_tile<EPI>(p, t);
        const bool kcm = RAGGED && !HALO && p.kc_major != nullptr &&
                         __ldg(p.kc_major + static_cast<int64_t>(c.n0) * p.ext_ld) != 0;
        if constexpr (HALO) {
          for (int kc = 0; kc < p.cin_blocks; ++kc, ++gp) {
            const int ps = gp % L::NP;
            mbar_wait(&pempty_bar[ps], ((gp / L::NP) & 1) ^ 1);
            mbar_expect_tx(&pfull_bar[ps], L::PATCH_DATA);
            tma_load_5d(patch + ps * L::PATCH_BYTES, &tmA, &pfull_bar[ps], 0, c.wo0 - 1, c.ho0 - 1, c.n0, kc * 8);
            for (int tap = 0; tap < 9; ++tap, ++g) {
              const int s = g % STAGES;
              mbar_wait(&empty_bar[s], ((g / STAGES) & 1) ^ 1);
              mbar_expect_tx(&full_bar[s], L::STAGE_BYTES);
              tma_load_2d(smem + s * L::STAGE_BYTES, &tmB, &full_bar[s], (tap * p.cin_blocks + kc) * 64, c.n_tile * BN);
            }
          }
        }
        for (int it = 0; !HALO && it < k_iters; ++it, ++g) {
          const int s = g % STAGES;
          mbar_wait(&empty_bar[s], ((g / STAGES) & 1) ^ 1);
          mbar_expect_tx(&full_bar[s], L::STAGE_BYTES);
          uint8_t* sa = smem + s * L::STAGE_BYTES;
          int tap = it / p.cin_blocks;
          int kc = it - tap * p.cin_blocks;
          int kb = it;                                // weight block of this k-iteration
          if (kcm) {                                  // HALO order: channel block outer, tap inner
            kc = it / p.taps;
            tap = it - kc * p.taps;
            kb = tap * p.cin_blocks + kc;
          }
          if (EPI == PERS_EPI_F32) {
            const int part = it / p.k_per_part;
            const int kk = it - part * p.k_per_part;
            // small cross terms first, (hi, hi) last: the tensor core's fp32 accumulation truncates, an error that grows
            // with the accumulator's magnitude per step - the 2/3 of the steps that add 2^-11-sized terms then run
            // while the accumulator is still small
            tma_load_2d(sa, part == 1 ? &tmR : &tmA, &full_bar[s], kk * 64, c.m_tile * 128);
            tma_load_2d(sa + L::A_BYTES, part == 0 ? &tmO : &tmB, &full_bar[s], kk * 64, c.n_tile * BN);
            continue;
          }
          if (p.k_split > 0 && it >= p.k_split) {
            tma_load_4d(sa, &tmR, &full_bar[s], (it - p.k_split) * 64, c.wo0 * p.a2_stride, c.ho0 * p.a2_stride, c.n0);
          } else if (p.a_spatial) {
            const int kh = tap / p.kw_taps;
            const int kw = tap - kh * p.kw_taps;
            tma_load_4d(sa, &tmA, &full_bar[s], kc * 64, c.wo0 * p.stride + kw - p.pad,
                        c.ho0 * p.stride + kh - p.pad, c.n0);
          } else {
            tma_load_2d(sa, &tmA, &full_bar[s], it * 64, pers_list_epi<EPI>() ? c.a_row : c.m_tile * 128);
          }
          tma_load_2d(sa + L::A_BYTES, &tmB, &full_bar[s], kb * 64, pers_list_epi<EPI>() ? c.b_row : c.n_tile * BN);
        }
      }
    }
    return;
  }

  // ---------------------------------------------------------------- consumers
  if constexpr (PP) setmaxnreg_inc<232>();         // the whole 128 x BN accumulator tile lives in each warpgroup
  // cooperative: accumulator rows 64*wg ..; ping-pong: the CTA-local tiles i with i & 1 == wg, all 128 rows
  const int wg = (warp >> 2) - 1;
  const int ctid = static_cast<int>(threadIdx.x) - 128;
  const bool leader = PP ? (ctid & 127) == 0 : ctid == 0;   // issues the residual loads and the output stores
  const int half0 = PP ? 0 : wg;                   // first 64-row half of the tile in this warpgroup's accumulators
  const int r0 = half0 * 64 + (warp & 3) * 16 + (lane >> 2);   // this thread's rows: r0 + 64 * half and + 8
  const int t4 = lane & 3;
  // invariant 4: per-warpgroup staging buffers, residual barrier and named barrier (ID 0 is __syncthreads)
  uint8_t* stg_w = stg + (PP ? wg * L::WG_STG_BYTES : 0);
  uint64_t* res_w = res_bar + (PP ? wg : 0);
  const int epi_bar = PP ? 1 + wg : 1;
  const int epi_threads = PP ? 128 : PERS_CONSUMER_THREADS;
  float acc[NH][BN / 2];
#pragma unroll
  for (int h = 0; h < NH; ++h)
#pragma unroll
    for (int j = 0; j < BN / 2; ++j) acc[h][j] = 0.f;

  uint32_t g = 0, i = PP ? wg : 0, gp = 0;
  for (int t = blockIdx.x + (PP ? wg * static_cast<int>(gridDim.x) : 0); t < p.total_tiles;
       t += (PP ? 2 : 1) * gridDim.x, i += PP ? 2 : 1) {
    const TileCoord c = decode_any_tile<EPI>(p, t);
    const uint32_t jw = PP ? i >> 1 : i;             // tiles this warpgroup has finished: the residual barrier's phase
    // ragged batches: bit 2 * hf + h = this thread's row r0 + 64 * hf + 8 * h lies inside its image (decided before the
    // main loop, where the previous tile's accumulators are dead)
    uint32_t keep = 0;
#pragma unroll
    for (int hf = 0; hf < NH; ++hf)
#pragma unroll
      for (int h = 0; h < 2; ++h)
        if (!RAGGED || row_in_extent(p, c.m_tile, c.wo0, c.ho0, c.n0, r0 + 64 * hf + 8 * h)) keep |= 1u << (2 * hf + h);
    if (EPI == PERS_EPI_CONV && p.has_res && leader) {
      // the residual tile goes into the staging buffers once the previous tile's stores have finished reading them
      // (bulk groups belong to the thread that committed them: each warpgroup's leader waits for its own stores)
      bulk_wait_read<0>();
      mbar_expect_tx(res_w, CHUNKS * L::STG_CHUNK);
      for (int ch = 0; ch < CHUNKS; ++ch) {
        if (p.a_spatial)
          tma_load_4d(stg_w + ch * L::STG_CHUNK, &tmR, res_w, c.n_tile * BN + ch * 64, c.wo0, c.ho0, c.n0);
        else
          tma_load_2d(stg_w + ch * L::STG_CHUNK, &tmR, res_w, c.n_tile * BN + ch * 64, c.m_tile * 128);
      }
    }
    if constexpr (PP) {
      // invariant 2: this tile's first ring (and patch) slot; every tile has k_iters = taps * cin_blocks k-iterations
      g = i * static_cast<uint32_t>(k_iters);
      gp = i * static_cast<uint32_t>(p.cin_blocks);
      // invariant 1: the partner warpgroup has passed every full-barrier wait of tile i - 1
      if (i > 0) mbar_wait(&mma_done[wg ^ 1], ((i - 1) >> 1) & 1);
    }

    // ------------------------------------------------------------ main loop
    if constexpr (HALO) {
      // K order: channel block outer, tap inner.  Output row r = 8 * ih + iw reads patch pixel (ih + kh) * HALO_W + iw + kw:
      // the 8 rows of a core matrix are consecutive pixels (16 B apart in a chunk), 8-row groups HALO_W pixels apart.
      bool prev_last = false;                       // the previous wgmma group was the last tap of its patch
      for (int kc = 0; kc < p.cin_blocks; ++kc, ++gp) {
        const int ps = gp % L::NP;
        mbar_wait(&pfull_bar[ps], (gp / L::NP) & 1);
        const uint32_t pa = smem_u32(patch + ps * L::PATCH_BYTES);
        for (int tap = 0; tap < 9; ++tap, ++g) {
          const int s = g % STAGES;
          const int kh = tap / 3, kw = tap - 3 * (tap / 3);
          mbar_wait(&full_bar[s], (g / STAGES) & 1);
          uint64_t adesc[NH];
#pragma unroll
          for (int h = 0; h < NH; ++h)
            adesc[h] = gmma_desc_noswizzle(pa + (((half0 + h) * 8 + kh) * HALO_W + kw) * 16, L::PATCH_CHUNK, HALO_W * 16);
          const uint64_t bdesc = gmma_desc_sw128(smem_u32(smem + s * L::STAGE_BYTES));
#pragma unroll
          for (int h = 0; h < NH; ++h)
#pragma unroll
            for (int j = 0; j < BN / 2; ++j) fence_operand(acc[h][j]);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < 4; ++k)
#pragma unroll
            for (int h = 0; h < NH; ++h)
              wgmma_f16<BN>(acc[h], adesc[h] + ((2 * k * L::PATCH_CHUNK) >> 4), bdesc + 2 * k, (kc | tap | k) != 0);
          wgmma_commit();
          wgmma_wait<1>();                          // the previous group is done: hand back its weight slot (and patch)
#pragma unroll
          for (int h = 0; h < NH; ++h)
#pragma unroll
            for (int j = 0; j < BN / 2; ++j) fence_operand(acc[h][j]);
          if ((kc | tap) != 0 && (ctid & 127) == 0) {
            mbar_arrive(&empty_bar[(g - 1) % STAGES]);
            if (prev_last) mbar_arrive(&pempty_bar[(gp - 1) % L::NP]);
          }
          prev_last = tap == 8;
        }
      }
      if (PP && lane == 0) mbar_arrive(&mma_done[wg]);   // this warp is done waiting: the partner may start
      wgmma_wait<0>();
#pragma unroll
      for (int h = 0; h < NH; ++h)
#pragma unroll
        for (int j = 0; j < BN / 2; ++j) fence_operand(acc[h][j]);
      if ((ctid & 127) == 0) {
        mbar_arrive(&empty_bar[(g - 1) % STAGES]);
        mbar_arrive(&pempty_bar[(gp - 1) % L::NP]);
      }
    }
    for (int it = 0; !HALO && it < k_iters; ++it, ++g) {
      const int s = g % STAGES;
      mbar_wait(&full_bar[s], (g / STAGES) & 1);
      const uint32_t sa = smem_u32(smem + s * L::STAGE_BYTES);
      uint64_t adesc[NH];
#pragma unroll
      for (int h = 0; h < NH; ++h) adesc[h] = gmma_desc_sw128(sa + (half0 + h) * 64 * 128);
      const uint64_t bdesc = gmma_desc_sw128(sa + L::A_BYTES);
#pragma unroll
      for (int h = 0; h < NH; ++h)
#pragma unroll
        for (int j = 0; j < BN / 2; ++j) fence_operand(acc[h][j]);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k)
#pragma unroll
        for (int h = 0; h < NH; ++h) wgmma_f16<BN>(acc[h], adesc[h] + 2 * k, bdesc + 2 * k, (it | k) != 0);
      wgmma_commit();
      wgmma_wait<1>();                              // the previous slot's MMAs are done: hand it back
#pragma unroll
      for (int h = 0; h < NH; ++h)
#pragma unroll
        for (int j = 0; j < BN / 2; ++j) fence_operand(acc[h][j]);
      if (it > 0 && (ctid & 127) == 0) mbar_arrive(&empty_bar[(g - 1) % STAGES]);
    }
    if constexpr (!HALO) {
      if (PP && lane == 0) mbar_arrive(&mma_done[wg]);   // this warp is done waiting: the partner may start
      wgmma_wait<0>();
#pragma unroll
      for (int h = 0; h < NH; ++h)
#pragma unroll
        for (int j = 0; j < BN / 2; ++j) fence_operand(acc[h][j]);
      if (k_iters > 0 && (ctid & 127) == 0) mbar_arrive(&empty_bar[(g - 1) % STAGES]);
    }

    // ------------------------------------------------------------ epilogue
    if (EPI == PERS_EPI_CONV) {
      if (p.has_res) {
        mbar_wait(res_w, jw & 1);                   // residual tile has landed in the staging buffers
      } else {
        if (leader) bulk_wait_read<0>();            // the previous tile's stores have left the staging buffers
        named_bar_sync(epi_bar, epi_threads);
      }
      conv_epilogue_to_staging<BN, NH, RAGGED>(acc, smem_u32(stg_w), r0, t4, p.scale + c.n_tile * BN,
                                               p.shift + c.n_tile * BN, p.has_res, p.relu, keep);
      fence_proxy_async_smem();                     // generic-proxy smem writes -> visible to the TMA engine
      named_bar_sync(epi_bar, epi_threads);
      if (leader) {
        for (int ch = 0; ch < CHUNKS; ++ch) {
          const int col0 = c.n_tile * BN + ch * 64;
          if (p.a_spatial) tma_store_4d(&tmO, stg_w + ch * L::STG_CHUNK, col0, c.wo0, c.ho0, c.n0);
          else tma_store_2d(&tmO, stg_w + ch * L::STG_CHUNK, col0, c.m_tile * 128);
        }
        bulk_commit();
      }
    } else {
      // ---------------------------------------------------------- similarity / whitening epilogues: row = query
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int64_t qi = static_cast<int64_t>(c.m_tile) * 128 + r0 + 8 * h;
        const bool valid = qi < p.M;
        if (EPI == PERS_EPI_SIM_FILTER || EPI == PERS_EPI_SIM_JOIN || EPI == PERS_EPI_SIM_FILTER_ALLOW) {
          // every match of the row (score >= the query's threshold) is appended to its candidate list: the four threads
          // holding a row reserve their slots with ONE atomicAdd and split them by a prefix sum over the quad.  The
          // self-join keeps only the columns after the row (col > row: the pair (i, j) once, i < j, never (i, i)).
          // The filtered search keeps only the columns whose allow bit is set: aw[g] holds the bits of the tile's
          // columns 32g .. 32g + 31, funnel-shifted out of the bitmap's words (allow_bit0 need not be a multiple of 32).
          constexpr bool JOIN = EPI == PERS_EPI_SIM_JOIN;
          constexpr bool ALLOW = EPI == PERS_EPI_SIM_FILTER_ALLOW;
          const float t_q = valid ? __ldg(p.thr + qi) : INFINITY;
          uint32_t aw[ALLOW ? BN / 32 : 1];
          if constexpr (ALLOW) {
            const int64_t b0 = p.allow_bit0 + static_cast<int64_t>(c.n_tile) * BN;   // bit of the tile's column 0
            const int64_t w_last = (p.allow_bit0 + p.N - 1) >> 5;                   // last word holding a row's bit
            const uint32_t* wq = p.allow + (valid ? qi : 0) * p.allow_ld;
            const int sh = static_cast<int>(b0 & 31);
            uint32_t lo = valid ? __ldg(wq + (b0 >> 5)) : 0u;
#pragma unroll
            for (int g = 0; g < BN / 32; ++g) {
              const int64_t w = (b0 >> 5) + g + 1;
              const uint32_t hi = (valid && w <= w_last) ? __ldg(wq + w) : 0u;
              aw[g] = __funnelshift_r(lo, hi, sh);
              lo = hi;
            }
          }
          auto allowed = [&](int cl) { return !ALLOW || ((aw[ALLOW ? cl >> 5 : 0] >> (cl & 31)) & 1u); };
          int cnt = 0;
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
            const int col = c.n_tile * BN + j * 8 + 2 * t4;
            cnt += (acc[0][4 * j + 2 * h] >= t_q && col < p.N && (!JOIN || col > qi) && allowed(j * 8 + 2 * t4)) ? 1 : 0;
            cnt += (acc[0][4 * j + 2 * h + 1] >= t_q && col + 1 < p.N && (!JOIN || col + 1 > qi) && allowed(j * 8 + 2 * t4 + 1))
                       ? 1 : 0;
          }
          int incl = cnt;
#pragma unroll
          for (int d = 1; d < 4; d <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, incl, d, 4);
            if (t4 >= d) incl += y;
          }
          const int total = __shfl_sync(0xffffffffu, incl, 3, 4);
          int base = 0;
          if (t4 == 0 && total > 0) base = atomicAdd(p.cand_cnt + qi, total);
          base = __shfl_sync(0xffffffffu, base, 0, 4);
          if (cnt > 0) {
            int pos = base + incl - cnt;
            unsigned long long* dst = p.cand + qi * p.cand_cap;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const float v = acc[0][4 * j + 2 * h + e];
                const int col = c.n_tile * BN + j * 8 + 2 * t4 + e;
                if (v >= t_q && col < p.N && (!JOIN || col > qi) && allowed(j * 8 + 2 * t4 + e)) {
                  if (pos < p.cand_cap)
                    dst[pos] = (static_cast<unsigned long long>(__float_as_uint(v)) << 32) | static_cast<unsigned int>(col);
                  ++pos;
                }
              }
            }
          }
        } else if (EPI == PERS_EPI_SIM_GMAX) {
          // maximum of each group of 32 database rows: the k-th largest group maximum is a valid lower bound on
          // the k-th best score (k distinct rows reach it) and costs 1/32 of the dense write + select
#pragma unroll
          for (int gi = 0; gi < BN / 32; ++gi) {
            const int nb0 = c.n_tile * BN + gi * 32;
            float m = -INFINITY;
#pragma unroll
            for (int j = 4 * gi; j < 4 * gi + 4; ++j) {
              const int col = c.n_tile * BN + j * 8 + 2 * t4;
              m = (col < p.N) ? fmaxf(m, acc[0][4 * j + 2 * h]) : m;
              m = (col + 1 < p.N) ? fmaxf(m, acc[0][4 * j + 2 * h + 1]) : m;
            }
            m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
            m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
            if (t4 == 0 && valid && nb0 < p.N) p.dense[qi * p.dense_ld + (nb0 >> 5)] = m;
          }
        } else if (EPI == PERS_EPI_SIM_LFILTER) {
          // the filter over a list tile: the same quad-level reservation, the query through slot_q, the row through perm
          const int r = r0 + 8 * h;
          const bool ok = r < c.m_valid;
          const int q = ok ? __ldg(p.slot_q + c.a_row + r) : 0;
          const float t_q = ok ? __ldg(p.thr + q) : INFINITY;
          int cnt = 0;
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
            const int col = j * 8 + 2 * t4;
            cnt += (acc[0][4 * j + 2 * h] >= t_q && col < c.n_valid) ? 1 : 0;
            cnt += (acc[0][4 * j + 2 * h + 1] >= t_q && col + 1 < c.n_valid) ? 1 : 0;
          }
          int incl = cnt;
#pragma unroll
          for (int d = 1; d < 4; d <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, incl, d, 4);
            if (t4 >= d) incl += y;
          }
          const int total = __shfl_sync(0xffffffffu, incl, 3, 4);
          int base = 0;
          if (t4 == 0 && total > 0) base = atomicAdd(p.cand_cnt + q, total);
          base = __shfl_sync(0xffffffffu, base, 0, 4);
          if (cnt > 0) {
            int pos = base + incl - cnt;
            unsigned long long* dst = p.cand + static_cast<int64_t>(q) * p.cand_cap;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const float v = acc[0][4 * j + 2 * h + e];
                const int col = j * 8 + 2 * t4 + e;
                if (v >= t_q && col < c.n_valid) {
                  if (pos < p.cand_cap) {
                    const unsigned int row = static_cast<unsigned int>(__ldg(p.perm + c.b_row + col));
                    dst[pos] = (static_cast<unsigned long long>(__float_as_uint(v)) << 32) | row;
                  }
                  ++pos;
                }
              }
            }
          }
        } else if (EPI == PERS_EPI_SIM_LGMAX) {
          // group maxima of a list tile: groups of 32 list positions, numbered from the list's first row
          const int r = r0 + 8 * h;
          const bool ok = r < c.m_valid;
          const int64_t gb = ok ? __ldg(p.gbase + c.a_row + r) + static_cast<int64_t>(c.n_tile) * (BN / 32) : 0;
#pragma unroll
          for (int gi = 0; gi < BN / 32; ++gi) {
            float m = -INFINITY;
#pragma unroll
            for (int j = 4 * gi; j < 4 * gi + 4; ++j) {
              const int col = j * 8 + 2 * t4;
              m = (col < c.n_valid) ? fmaxf(m, acc[0][4 * j + 2 * h]) : m;
              m = (col + 1 < c.n_valid) ? fmaxf(m, acc[0][4 * j + 2 * h + 1]) : m;
            }
            m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
            m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
            if (t4 == 0 && ok && gi * 32 < c.n_valid) p.dense[gb + gi] = m;
          }
        } else if (valid) {                           // PERS_EPI_SIM_DENSE / PERS_EPI_F32
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
            const int col = c.n_tile * BN + j * 8 + 2 * t4;
            if (col >= p.N) continue;
            float v0 = acc[0][4 * j + 2 * h], v1 = acc[0][4 * j + 2 * h + 1];
            if (EPI == PERS_EPI_F32 && p.scale != nullptr) {
              v0 *= __ldg(p.scale + col);
              if (col + 1 < p.N) v1 *= __ldg(p.scale + col + 1);
            }
            store_dense_pair(p, qi, col, v0, v1);
          }
        }
      }
    }
  }
  if (EPI == PERS_EPI_CONV && leader) bulk_wait<0>();     // all output bytes written before the CTA retires
}

template <int BN, int STAGES, int EPI, bool HALO = false, bool RAGGED = false, bool PP = false>
int conv_pers_launch(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmR, const CUtensorMap& tmO,
                     const ConvPersParams& p, int num_sms, cudaStream_t stream) {
  using L = ConvPersSmem<BN, STAGES, EPI, HALO, PP>;
  static_assert(L::TOTAL <= 232448, "shared memory budget exceeded");
  auto kern = conv_pers_kernel<BN, STAGES, EPI, HALO, RAGGED, PP>;
  static std::atomic<uint64_t> attr_done{0};
  if (first_launch_on_device(attr_done))
    DIRB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L::TOTAL));
  const int grid = p.total_tiles < num_sms ? p.total_tiles : num_sms;
  DIRB_CUDA(launch_pdl(kern, dim3(grid), dim3(PERS_THREADS), L::TOTAL, stream, tmA, tmB, tmR, tmO, p));
  count_launch();
  return 0;
}

}  // namespace dirb
