// Similarity + top-k over one row shard of the descriptor database.
//
// Replaces the reference's dense  scores = matmul(q, db)  (dirtorch/utils/common.py:30-38, test_dir.py:145) +
// per-query sort (datasets/generic.py:207,221) for the first k ranks, without materialising the Q x N matrix:
//
//   1. queries -> fp16, counters / retry gates / status cleared                    (search_prep_kernel)
//   2. seed:   wgmma GEMM of the queries against the first S rows.  The epilogue keeps the maximum of every group
//              of 32 consecutive rows (PERS_EPI_SIM_GMAX; 1/32 of the dense score traffic); per query the k-th largest
//              group maximum t_S has >= k rows at or above it, so it is a lower bound on the final k-th score.
//              (fewer than k groups: dense scores, PERS_EPI_SIM_DENSE)                 (kth_dense_kernel)
//   3. filter: wgmma GEMM against all N rows; the epilogue appends (score,row) to the query's candidate list
//              only when score >= t_S - 2*eps16                                     (PERS_EPI_SIM_FILTER)
//      (for N <= S step 3 is a scan of the dense scores instead: dense_compact_kernel)
//   4. select: exact k-th largest candidate score t (radix select, cand_kth_kernel).  A query whose list overflowed
//              gets a tighter threshold from what was captured and raises a device-side gate; the (always enqueued)
//              retry passes of steps 3-4 return at once unless their gate is up - no host round trip.
//   5. finish: survivors = candidates with score >= t - 2*eps16, exact re-scoring (fp64 accumulation of the fp32
//              rows) and sort (score desc, index asc), one launch, one block per query      (search_finish_kernel)
// The only host synchronisation is the status check at the very end (overflow that the retries could not resolve);
// with option deferred_check it moves to dirb200_index_check / the start of the next search.
//
// eps16 bounds |fp16-path score - exact score| (unit-norm rows: 2 * 2^-11 from the operand roundings + fp32
// accumulation, default 1.2e-3); any row of the true top-k then satisfies the step-3 and step-4 conditions, so the
// result is the exact top-k (same argument twice).  Candidate-buffer overflow raises the threshold from what was
// captured and re-runs the filter pass.  With several shards the phases are split (search_begin / search_finish)
// so that the caller can MIN-reduce the per-shard selection thresholds in between (see cand_kth_kernel).
// The GEMMs run on the persistent warp-specialised kernel of conv_pers.cuh (128 x 128 tiles, K = D).
// Filtered search (an allow bitmap attached with dirb200_index_set_allow, DESIGN.md section 4.13, rules F1-F6): the seed
// rows are the first S rows allowed for every query of the block, gathered into a buffer of their own (allow_and_kernel,
// allow_seed_rows_kernel, allow_gather_kernel, allow_kth_kernel), and the filter pass tests each column's bit
// (PERS_EPI_SIM_FILTER_ALLOW; always the GEMM pass, never the dense scan of step 3).  Steps 4-5 are unchanged.
#include <math.h>

#include <limits.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <string>
#include <vector>

#include "block.cuh"
#include "conv.h"
#include "conv_pers.cuh"
#include "exact_dot.cuh"
#include "label_count.h"

namespace dirb {
namespace {

constexpr int SEL_THREADS = 512;

struct DenseAcc {
  const float* p;
  __device__ float operator()(int i) const { return p[i]; }
};
struct CandAcc {
  const unsigned long long* p;
  __device__ float operator()(int i) const { return __uint_as_float(static_cast<uint32_t>(p[i] >> 32)); }
};

// k-th largest of n values (block_radix_kth on f2key). n < k -> -inf.
template <class Acc>
__device__ float block_kth_largest(Acc acc, int n, int k, uint32_t* hist /*[256]*/, uint32_t* bc /*[2]*/) {
  if (n < k) return -INFINITY;
  return key2f(block_radix_kth<uint32_t>([&](int i) { return f2key(acc(i)); }, n, k, hist, bc));
}

// thr[q] = (k-th largest of dense[q][0..S)) - band; k2 > 0: also thr2[q] = (k2-th largest) - band (the seed bound a shard
// contributes to the MIN over the shards, see dirb200_index_search_sharded).
__global__ void __launch_bounds__(SEL_THREADS) kth_dense_kernel(const float* __restrict__ dense, int64_t ld, int S,
                                                                int k, float band, float* __restrict__ thr, int k2,
                                                                float* __restrict__ thr2) {
  __shared__ uint32_t hist[256];
  __shared__ uint32_t bc[2];
  const int q = blockIdx.x;
  const float t = block_kth_largest(DenseAcc{dense + q * ld}, S, k, hist, bc);
  if (threadIdx.x == 0) thr[q] = t - band;
  if (k2 > 0) {
    __syncthreads();
    const float t2 = (k2 == k) ? t : block_kth_largest(DenseAcc{dense + q * ld}, S, k2, hist, bc);
    if (threadIdx.x == 0) thr2[q] = t2 - band;
  }
}

// N <= S: candidates straight from the dense scores.
__global__ void dense_compact_kernel(const float* __restrict__ dense, int64_t ld, int N, const float* __restrict__ thr,
                                     unsigned long long* __restrict__ cand, int* __restrict__ cnt, int cap,
                                     const int* __restrict__ gate) {
  if (gate != nullptr && *reinterpret_cast<const volatile int*>(gate) == 0) return;
  const int q = blockIdx.y;
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  const float v = dense[q * ld + n];
  if (v >= thr[q]) {
    const int pos = atomicAdd(cnt + q, 1);
    if (pos < cap)
      cand[static_cast<int64_t>(q) * cap + pos] = (static_cast<unsigned long long>(__float_as_uint(v)) << 32) | static_cast<unsigned>(n);
  }
}

// Status block of a search (device, 8 x u64; copied to pinned host memory at the end of phase 2):
//   [0] error bits: 1 = candidate overflow left after the last retry pass, 2 = more than cap2 survivors for some query
//   [1] candidates captured (sum over queries)   [2] survivors re-scored   [3] retry passes that actually ran
enum { ST_ERR = 0, ST_CAND = 1, ST_SURV = 2, ST_RETRIES = 3, ST_WORDS = 8 };

// Per query: exact k-th and k_shard-th largest candidate scores (fp16-path scores).
//   kth_k[q]  : local k-th best - always a valid lower bound on the global k-th best
//   sel[q]    : local min(k_shard, N)-th best; the MINIMUM of this value over all shards is a valid and much tighter
//               lower bound on the global k-th best as long as the shards certify k rows between them,
//               sum_g min(k_shard, N_g) >= min(k, N_total) (shard g holds min(k_shard, N_g) rows at or above its own
//               value) - the caller picks k_shard accordingly (ceil(k / shards) for evenly filled shards, see
//               dist.py: shard_quota) and min-reduces sel.
// Overflow (cnt > cap) is resolved on the device: the query's list is emptied, the tighter threshold
// kth(captured) - band goes to thr[q] and gate_out[0] is raised, which arms the next (gated) filter pass + selection;
// finished queries get thr[q] = +inf so that a re-run leaves them alone.  `gate_in` != nullptr: this launch is itself
// such a retry pass and returns at once unless *gate_in != 0.  `last` = no further retry follows: a remaining
// overflow becomes error bit 1.
__global__ void __launch_bounds__(SEL_THREADS) cand_kth_kernel(const unsigned long long* __restrict__ cand,
                                                               int* __restrict__ cnt, int cap, int k, int k_shard,
                                                               float band, float* __restrict__ kth_k,
                                                               float* __restrict__ sel, float* __restrict__ thr,
                                                               int64_t n_rows, const int* __restrict__ gate_in,
                                                               int* __restrict__ gate_out, int last,
                                                               unsigned long long* __restrict__ status) {
  __shared__ uint32_t hist[256];
  __shared__ uint32_t bc[2];
  if (gate_in != nullptr && *reinterpret_cast<const volatile int*>(gate_in) == 0) return;
  const int q = blockIdx.x;
  if (gate_in != nullptr && q == 0 && threadIdx.x == 0) atomicAdd(status + ST_RETRIES, 1ull);
  const int total = cnt[q];
  const int n = min(total, cap);
  const float thr_in = thr[q];                 // what the filter pass used: (a lower bound on the global k-th best) - band
  const unsigned long long* c = cand + static_cast<int64_t>(q) * cap;
  const int kk = (n_rows < static_cast<int64_t>(k)) ? static_cast<int>(n_rows) : k;
  const float t = block_kth_largest(CandAcc{c}, n, kk, hist, bc);
  if (total > cap) {
    if (threadIdx.x == 0) {
      if (last) {
        atomicOr(status + ST_ERR, 1ull);
        kth_k[q] = INFINITY;      // no survivors for this query; the error is reported by the status check
        sel[q] = INFINITY;
        thr[q] = INFINITY;
      } else {
        thr[q] = t - band;
        cnt[q] = 0;               // the retry pass refills the list from scratch
        *gate_out = 1;
      }
    }
    return;
  }
  float ts = t;
  if (k_shard < kk) {
    __syncthreads();
    ts = block_kth_largest(CandAcc{c}, n, k_shard, hist, bc);
  }
  // Fewer than k_shard rows above a filter threshold that came from the other shards: this shard's k_shard-th best lies
  // below that bound, which is itself a valid lower bound on the global k-th best - report the bound instead of -inf
  // (the MIN over the shards must stay selective).  Shards with fewer than k_shard ROWS report their worst row.
  if (ts == -INFINITY && n_rows >= static_cast<int64_t>(k_shard) && thr_in != -INFINITY) ts = thr_in + band;
  if (threadIdx.x == 0) {
    kth_k[q] = t;
    sel[q] = ts;
    thr[q] = INFINITY;
  }
}

// Start of a search: queries -> fp16 (the A operand of the tensor-core passes), candidate counters, retry gates and
// the status block cleared.  One launch instead of a conversion kernel + memsets.
__global__ void search_prep_kernel(const float* __restrict__ q32, __half* __restrict__ q16, int64_t n, int* __restrict__ cnt,
                                   int Q, int* __restrict__ gates, int n_gates, unsigned long long* __restrict__ status) {
  const int64_t gtid = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  const int64_t i = gtid * 4;
  if (i + 3 < n) {
    const float4 v = *reinterpret_cast<const float4*>(q32 + i);
    uint2 o;
    o.x = pack_h2(v.x, v.y);
    o.y = pack_h2(v.z, v.w);
    *reinterpret_cast<uint2*>(q16 + i) = o;
  } else {
    for (int64_t j = i; j < n; ++j) q16[j] = __float2half_rn(q32[j]);
  }
  if (gtid < Q) cnt[gtid] = 0;
  if (gtid < n_gates) gates[gtid] = 0;
  if (gtid < ST_WORDS) status[gtid] = 0ull;
}

// Empty shard: nothing can be selected (+inf never lowers the MIN over the shards) / nothing to return.
__global__ void fill_f32_kernel(float* __restrict__ p, int n, float v) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}
__global__ void fill_empty_result_kernel(double* __restrict__ sc, int64_t* __restrict__ ix, int64_t n) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i < n) {
    sc[i] = -INFINITY;
    ix[i] = -1;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Seed of the filtered search (rule F2).  The allow bitmap is in global row numbering: local row r of this shard is bit
// bit0 + r of a query's row of words (ld words apart; ld = 0: one row shared by every query).
// iw[j] = AND over the nrow bitmap rows of the bits of local rows 32j .. 32j + 31 (rows >= N cleared).
__global__ void allow_and_kernel(const uint32_t* __restrict__ allow, int64_t ld, int64_t bit0, int nrow, int64_t N,
                                 uint32_t* __restrict__ iw) {
  const int64_t j = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (j >= (N + 31) >> 5) return;
  const int64_t b = bit0 + 32 * j, w = b >> 5;
  const int sh = static_cast<int>(b & 31);
  const bool two = sh != 0 && (w + 1) * 32 < bit0 + N;      // the window spans two words
  uint32_t v = 0xffffffffu;
#pragma unroll 4
  for (int q = 0; q < nrow; ++q) {
    const uint32_t* a = allow + q * ld;
    v &= __funnelshift_r(__ldg(a + w), two ? __ldg(a + w + 1) : 0u, sh);
  }
  const int64_t rem = N - 32 * j;
  if (rem < 32) v &= (1u << rem) - 1u;
  iw[j] = v;
}

// The first S set bits of iw[0 .. W) in row order -> rows[0 .. n), *n_out = n = min(popcount, S).  One block; each thread
// takes four words per step, and the block's popcounts are placed by one block_scan.
constexpr int ALLOW_SCAN_THREADS = 1024;
__global__ void __launch_bounds__(ALLOW_SCAN_THREADS) allow_seed_rows_kernel(const uint32_t* __restrict__ iw, int64_t W, int S,
                                                                             int* __restrict__ rows, int* __restrict__ n_out) {
  __shared__ int warp_sums[ALLOW_SCAN_THREADS / 32];
  int base = 0;
  for (int64_t w0 = 0; w0 < W && base < S; w0 += 4 * ALLOW_SCAN_THREADS) {
    const int64_t j0 = w0 + 4 * static_cast<int64_t>(threadIdx.x);
    uint32_t bits[4];
    int cnt = 0;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      bits[e] = j0 + e < W ? __ldg(iw + j0 + e) : 0u;
      cnt += __popc(bits[e]);
    }
    int total;
    int pos = base + block_scan(cnt, warp_sums, &total) - cnt;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      uint32_t m = bits[e];
      while (m != 0u && pos < S) {
        rows[pos++] = static_cast<int>(32 * (j0 + e)) + __ffs(m) - 1;
        m &= m - 1u;
      }
    }
    base += total;                                 // the same on every thread: the loop ends for the whole block
  }
  if (threadIdx.x == 0) *n_out = min(base, S);
}

// seed16[p] = db16[rows[p]] for p < *n_seed (one warp per row, 16-byte copies); the rows past it are not written.
__global__ void allow_gather_kernel(const __half* __restrict__ db16, int D, const int* __restrict__ rows,
                                    const int* __restrict__ n_seed, int S, __half* __restrict__ seed16) {
  const int p = static_cast<int>((blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (p >= S || p >= *n_seed) return;
  const uint4* src = reinterpret_cast<const uint4*>(db16 + static_cast<int64_t>(__ldg(rows + p)) * D);
  uint4* dst = reinterpret_cast<uint4*>(seed16 + static_cast<int64_t>(p) * D);
  for (int i = lane; i < D / 8; i += 32) dst[i] = __ldg(src + i);
}

// kth_dense_kernel over the gathered seed rows: only the first *n_seed of the S rows hold allowed rows.  Group maxima
// (gmax) count the full groups of 32 of them (all S rows valid: every group, the last one clipped by the GEMM itself);
// fewer than k values give -inf (rule F2: no allowed row is certified).
__global__ void __launch_bounds__(SEL_THREADS) allow_kth_kernel(const float* __restrict__ dense, int64_t ld, int S, int gmax,
                                                                const int* __restrict__ n_seed, int k, float band,
                                                                float* __restrict__ thr, int k2, float* __restrict__ thr2) {
  __shared__ uint32_t hist[256];
  __shared__ uint32_t bc[2];
  const int q = blockIdx.x;
  const int n = *n_seed;
  const int n_vals = !gmax ? n : (n == S ? (S + 31) / 32 : n / 32);
  const float t = block_kth_largest(DenseAcc{dense + q * ld}, n_vals, k, hist, bc);
  if (threadIdx.x == 0) thr[q] = t - band;
  if (k2 > 0) {
    __syncthreads();
    const float t2 = (k2 == k) ? t : block_kth_largest(DenseAcc{dense + q * ld}, n_vals, k2, hist, bc);
    if (threadIdx.x == 0) thr2[q] = t2 - band;
  }
}

// Clear bit rows[i] of bitmap row q for every i in [off[q], off[q + 1]) (rows outside [0, 32 ld) are skipped).
// atomicAnd: the result does not depend on the order, and a row listed twice is cleared once.
__global__ void allow_exclude_kernel(uint32_t* __restrict__ words, int64_t ld, const int64_t* __restrict__ off,
                                     const int64_t* __restrict__ rows) {
  const int q = blockIdx.x;
  uint32_t* wq = words + q * ld;
  for (int64_t i = off[q] + threadIdx.x; i < off[q + 1]; i += blockDim.x) {
    const int64_t r = rows[i];
    if (r >= 0 && r < 32 * ld) atomicAnd(wq + (r >> 5), ~(1u << (r & 31)));
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Peer exchange of the sharded search (dirb200_index_search_sharded): the two collectives of the protocol - MIN of the
// per-shard selection thresholds, gather of the per-shard lists - are done by the producing kernels themselves with
// stores into the peers' memory over NVLink (P2P mappings, CUDA IPC between the one-process-per-GPU ranks), and the
// consuming kernels wait on flags in their OWN memory.  Every rank owns one exchange buffer of identical layout:
//   [0]   epoch (u32; the current search, bumped by the last block of the merge)      [16..] block-completion counters
//   [64]  flag_sel[2][8]   [128] flag_list[2][8]   [192] flag_seed[2][8]
//                                                    written by rank g into slot g of EVERY rank (release, system scope)
//   [256] sel[2][G][max_q], seed[2][G][max_q] fp32 | score[2][G][max_q*max_k] fp64 | idx[2][G][max_q*max_k] int64
// Slots are double-buffered by epoch parity: rank r overwrites parity p two searches later, after it has seen every peer's
// lists of the search in between - which a peer publishes only after its own merge of the earlier search has read them.
constexpr int X_MAXW = 8;
constexpr int X_OFF_EPOCH = 0, X_OFF_CNT = 16, X_OFF_FSEL = 64, X_OFF_FLIST = 128, X_OFF_FSEED = 192, X_OFF_SEL = 256;
constexpr int X_TAB_SEL = 0, X_TAB_SEED = 1;              // float tables [2][G][max_q]: selection thresholds, seed bounds
struct PeerX {
  int world, rank, max_q, max_k;      // world == 0: no exchange (plain single-shard kernels)
  uint8_t* peer[X_MAXW];              // every rank's exchange buffer as mapped in THIS process (peer[rank] = own)
};
__host__ __device__ inline size_t x_tab_bytes(int world, int max_q) { return (static_cast<size_t>(2) * world * max_q * 4 + 255) / 256 * 256; }
__host__ __device__ inline size_t x_sel_bytes(int world, int max_q) { return 2 * x_tab_bytes(world, max_q); }
__host__ __device__ inline size_t x_off_tab(int tab, int world, int max_q) { return X_OFF_SEL + tab * x_tab_bytes(world, max_q); }
__host__ __device__ inline size_t x_list_elems(int max_q, int max_k) { return static_cast<size_t>(max_q) * max_k; }
__host__ __device__ inline size_t x_off_score(int world, int max_q) { return X_OFF_SEL + x_sel_bytes(world, max_q); }
__host__ __device__ inline size_t x_off_idx(int world, int max_q, int max_k) {
  return x_off_score(world, max_q) + static_cast<size_t>(2) * world * x_list_elems(max_q, max_k) * 8;
}
__host__ __device__ inline size_t x_total_bytes(int world, int max_q, int max_k) {
  return x_off_idx(world, max_q, max_k) + static_cast<size_t>(2) * world * x_list_elems(max_q, max_k) * 8;
}

__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t x_epoch(const PeerX& x) {
  return *reinterpret_cast<const volatile uint32_t*>(x.peer[x.rank] + X_OFF_EPOCH);
}
// One thread: wait until every rank has published epoch e in this rank's flag row.  Bounded (~10 s): a peer that never
// arrives becomes error bit 4 of the status block instead of a hung GPU.
__device__ __forceinline__ void x_wait_flags(const PeerX& x, int flag_off, uint32_t e, unsigned long long* status) {
  const uint32_t* f = reinterpret_cast<const uint32_t*>(x.peer[x.rank] + flag_off) + (e & 1u) * X_MAXW;
  for (int g = 0; g < x.world; ++g) {
    uint32_t spins = 0;
    while (static_cast<int32_t>(ld_acquire_sys(f + g) - e) < 0) {
      __nanosleep(100);
      if (++spins > (1u << 26)) {
        if (status) atomicOr(status + ST_ERR, 4ull);
        break;
      }
    }
  }
}
// End of a producing kernel: the LAST block to get here publishes epoch e in slot `rank` of every rank's flag row.
__device__ __forceinline__ void x_signal_when_all_blocks_done(const PeerX& x, int cnt_slot, int flag_off, uint32_t e) {
  __threadfence_system();                                   // this thread's stores to the peers before its block's arrival
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned int* cnt = reinterpret_cast<unsigned int*>(x.peer[x.rank] + X_OFF_CNT) + cnt_slot;
    if (atomicAdd(cnt, 1u) == gridDim.x * gridDim.y - 1u) {
      *cnt = 0u;
      __threadfence_system();
      for (int g = 0; g < x.world; ++g)
        st_release_sys(reinterpret_cast<uint32_t*>(x.peer[g] + flag_off) + (e & 1u) * X_MAXW + x.rank, e);
    }
  }
}

// This shard's per-query values (seed bounds / selection thresholds) into slot `rank` of every rank's float table.
__global__ void tab_push_kernel(PeerX x, const float* __restrict__ local, int Q, int tab, int flag_off, int cnt_slot) {
  const uint32_t e = x_epoch(x);
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q < Q) {
    const float v = local[q];
    const size_t o = x_off_tab(tab, x.world, x.max_q) + ((static_cast<size_t>(e & 1u) * x.world + x.rank) * x.max_q + q) * 4;
    for (int g = 0; g < x.world; ++g) *reinterpret_cast<float*>(x.peer[g] + o) = v;
  }
  x_signal_when_all_blocks_done(x, cnt_slot, flag_off, e);
}

// MIN over the shards of one float table, per query (waits for every rank's flag).
__device__ __forceinline__ float x_tab_min(const PeerX& x, int tab, uint32_t epoch, int q) {
  const float* t = reinterpret_cast<const float*>(x.peer[x.rank] + x_off_tab(tab, x.world, x.max_q)) +
                   static_cast<size_t>(epoch & 1u) * x.world * x.max_q;
  float m = INFINITY;
  for (int g = 0; g < x.world; ++g) m = fminf(m, __ldcg(t + static_cast<size_t>(g) * x.max_q + q));
  return m;
}

// Filter threshold of the sharded search: thr[q] = max(local k-th seed bound, MIN over the shards of their c-th seed
// bounds).  Both are lower bounds on the global k-th best score (the second by the shard-quota argument: every shard
// certifies c rows at or above its own value, G * c >= k), and the second is ~10x more selective on a G = 8 split:
// the local one keeps ~k / S of the rows as candidates, the global one ~c / S.
__global__ void thr_min_kernel(PeerX x, float* __restrict__ thr, int Q, unsigned long long* status) {
  const uint32_t e = x_epoch(x);
  if (threadIdx.x == 0) x_wait_flags(x, X_OFF_FSEED, e, status);
  __syncthreads();
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q < Q) thr[q] = fmaxf(thr[q], x_tab_min(x, X_TAB_SEED, e, q));
}

// Phase 2 of a search in ONE launch, one block per query:
//   survivors = candidates with fp16-path score >= max(sel[q], kth_k[q]) - band   (compacted into shared memory)
//   exact score of each survivor = fp64-accumulated dot product of the fp32 rows  (one warp per survivor)
//   bitonic sort by (score desc, row asc), first k written as (fp64 score, int64 global index).
// Replaces three launches whose grids were sized for the worst case (cap2 survivors per query) although a shard of a
// G-way split keeps only ~1.4 k / G rows per query.
constexpr int FIN_THREADS = 512;
__global__ void __launch_bounds__(FIN_THREADS) search_finish_kernel(
    const unsigned long long* __restrict__ cand, const int* __restrict__ cnt, int cap, const float* __restrict__ kth_k,
    const float* __restrict__ sel, float band, const float* __restrict__ q32, const float* __restrict__ db32, int D,
    int cap2, int64_t offset, int k, double* __restrict__ out_score, int64_t* __restrict__ out_idx,
    unsigned long long* __restrict__ status, const PeerX x) {
  // x.world > 0 (sharded search over peer memory): the selection threshold is the MINIMUM over the shards of the values the
  // peers stored into this rank's sel table (waits for their flags), and the ordered list goes to slot `rank` of EVERY
  // rank's list table instead of out_score / out_idx - MIN all-reduce and all-gather fused into this kernel.
  extern __shared__ uint8_t sm[];
  __shared__ int s_n;
  __shared__ float s_sel;
  double* sc = reinterpret_cast<double*>(sm);          // [cap2]
  int* ix = reinterpret_cast<int*>(sc + cap2);         // [cap2]
  const int q = blockIdx.x;
  const int n = cnt ? min(cnt[q], cap) : 0;            // (empty shard: no candidate buffers at all)
  const unsigned long long* c = cand + static_cast<int64_t>(q) * cap;
  const uint32_t epoch = x.world > 0 ? x_epoch(x) : 0u;
  if (threadIdx.x == 0) {
    s_n = 0;
    if (x.world > 0) {
      x_wait_flags(x, X_OFF_FSEL, epoch, status);
      s_sel = x_tab_min(x, X_TAB_SEL, epoch, q);
    } else {
      s_sel = sel[q];
    }
  }
  __syncthreads();
  const float t2 = fmaxf(s_sel, kth_k ? kth_k[q] : INFINITY) - band;
  for (int i = threadIdx.x; i < n; i += FIN_THREADS) {
    const unsigned long long e = c[i];
    if (__uint_as_float(static_cast<uint32_t>(e >> 32)) >= t2) {
      const int pos = atomicAdd(&s_n, 1);
      if (pos < cap2) ix[pos] = static_cast<int>(e & 0xffffffffu);
    }
  }
  __syncthreads();
  const int found = s_n;
  const int ns = min(found, cap2);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int w = warp; w < ns; w += FIN_THREADS / 32) {
    const double acc = exact_dot_warp(q32 + static_cast<int64_t>(q) * D, db32 + static_cast<int64_t>(ix[w]) * D, D, lane);
    if (lane == 0) sc[w] = acc;
  }
  int P = 2;
  while (P < ns) P <<= 1;
  for (int i = ns + threadIdx.x; i < P; i += FIN_THREADS) {
    sc[i] = -INFINITY;
    ix[i] = INT_MAX;
  }
  __syncthreads();
  block_bitonic_sort<FIN_THREADS>(sc, ix, P,
                                  [](double sa, int ia, double sb, int ib) { return ranks_before(sa, ia, sb, ib); });
  if (x.world > 0) {
    const size_t slot = (static_cast<size_t>(epoch & 1u) * x.world + x.rank) * x_list_elems(x.max_q, x.max_k) + static_cast<size_t>(q) * k;
    const size_t o_sc = x_off_score(x.world, x.max_q) + slot * 8, o_ix = x_off_idx(x.world, x.max_q, x.max_k) + slot * 8;
    for (int i = threadIdx.x; i < k; i += FIN_THREADS) {
      const bool ok = i < ns;
      const double vs = ok ? sc[i] : -INFINITY;
      const int64_t vi = ok ? static_cast<int64_t>(ix[i]) + offset : -1;
      for (int g = 0; g < x.world; ++g) {
        reinterpret_cast<double*>(x.peer[g] + o_sc)[i] = vs;
        reinterpret_cast<int64_t*>(x.peer[g] + o_ix)[i] = vi;
      }
    }
  } else {
    for (int i = threadIdx.x; i < k; i += FIN_THREADS) {
      const bool ok = i < ns;
      out_score[static_cast<int64_t>(q) * k + i] = ok ? sc[i] : -INFINITY;
      out_idx[static_cast<int64_t>(q) * k + i] = ok ? static_cast<int64_t>(ix[i]) + offset : -1;
    }
  }
  if (threadIdx.x == 0) {
    if (found > cap2) atomicOr(status + ST_ERR, 2ull);
    atomicAdd(status + ST_CAND, static_cast<unsigned long long>(n));
    atomicAdd(status + ST_SURV, static_cast<unsigned long long>(ns));
  }
  if (x.world > 0) x_signal_when_all_blocks_done(x, 1, X_OFF_FLIST, epoch);
}

// Phase 2 for k > 1024 (the deep path).  The survivors, their exact scores (exact_dot_warp) and their order are those
// of search_finish_kernel, but they live in global memory and each step runs over many blocks per query:
//   deep_compact_kernel   survivors (fp16-path score >= max(sel, kth_k) - band) -> surv_row[q][cap2], surv_cnt[q]
//   deep_rescore_kernel   one warp per survivor: exact score -> surv_sc[q][cap2]
//   deep_run_sort_kernel  runs of SORT_RUN survivors bitonic-sorted in shared memory -> (score, global index) in place
//   merge_runs_kernel     rank-based merge of the sorted runs, first k entries (also dirb200_topk_merge at large G*k)
// The last two are sort_runs_merge.

__global__ void deep_compact_kernel(const unsigned long long* __restrict__ cand, const int* __restrict__ cnt, int cap,
                                    const float* __restrict__ kth_k, const float* __restrict__ sel, float band,
                                    int* __restrict__ surv_row, int* __restrict__ surv_cnt, int cap2,
                                    unsigned long long* __restrict__ status) {
  const int q = blockIdx.y;
  const int n = min(cnt[q], cap);
  const float t2 = fmaxf(sel[q], kth_k[q]) - band;
  const unsigned long long* c = cand + static_cast<int64_t>(q) * cap;
  const int lane = threadIdx.x & 31;
  const int n_round = (n + 31) & ~31;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_round; i += gridDim.x * blockDim.x) {
    bool keep = false;
    int row = 0;
    if (i < n) {
      const unsigned long long e = c[i];
      keep = __uint_as_float(static_cast<uint32_t>(e >> 32)) >= t2;
      row = static_cast<int>(e & 0xffffffffu);
    }
    const unsigned m = __ballot_sync(0xffffffffu, keep);
    int base = 0;
    if (lane == 0 && m) base = atomicAdd(surv_cnt + q, __popc(m));
    base = __shfl_sync(0xffffffffu, base, 0);
    if (keep) {
      const int pos = base + __popc(m & ((1u << lane) - 1u));
      if (pos < cap2) surv_row[static_cast<int64_t>(q) * cap2 + pos] = row;
      else atomicOr(status + ST_ERR, 2ull);
    }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) atomicAdd(status + ST_CAND, static_cast<unsigned long long>(n));
}

__global__ void deep_rescore_kernel(const float* __restrict__ q32, const float* __restrict__ db32, int D,
                                    const int* __restrict__ surv_row, const int* __restrict__ surv_cnt, int cap2,
                                    double* __restrict__ surv_sc) {
  const int q = blockIdx.y;
  const int ns = min(surv_cnt[q], cap2);
  const int wpb = blockDim.x >> 5, lane = threadIdx.x & 31;
  const int64_t o = static_cast<int64_t>(q) * cap2;
  for (int w = blockIdx.x * wpb + (threadIdx.x >> 5); w < ns; w += gridDim.x * wpb) {
    const double acc = exact_dot_warp(q32 + static_cast<int64_t>(q) * D, db32 + static_cast<int64_t>(surv_row[o + w]) * D, D, lane);
    if (lane == 0) surv_sc[o + w] = acc;
  }
}

// Block x sorts run x of query y by (score desc, row asc) and writes it back as (score, global index); the tail of the
// last run becomes (-inf, -1), which the merge treats as empty.  Runs past the survivor count are never read.
__global__ void __launch_bounds__(FIN_THREADS) deep_run_sort_kernel(const int* __restrict__ surv_row,
                                                                    const int* __restrict__ surv_cnt, int cap2,
                                                                    int64_t offset, double* __restrict__ surv_sc,
                                                                    int64_t* __restrict__ run_ix,
                                                                    unsigned long long* __restrict__ status) {
  __shared__ double sc[SORT_RUN];
  __shared__ int ix[SORT_RUN];
  const int q = blockIdx.y;
  const int ns = min(surv_cnt[q], cap2);
  const int base = blockIdx.x * SORT_RUN;
  if (base >= ns) return;                                  // uniform over the block
  const int n = min(SORT_RUN, ns - base);
  const int64_t o = static_cast<int64_t>(q) * cap2 + base;
  int P = 2;
  while (P < n) P <<= 1;
  for (int i = threadIdx.x; i < P; i += FIN_THREADS) {
    const bool ok = i < n;
    sc[i] = ok ? surv_sc[o + i] : -INFINITY;
    ix[i] = ok ? surv_row[o + i] : INT_MAX;
  }
  __syncthreads();
  block_bitonic_sort<FIN_THREADS>(sc, ix, P,
                                  [](double sa, int ia, double sb, int ib) { return ranks_before(sa, ia, sb, ib); });
  for (int i = threadIdx.x; i < SORT_RUN; i += FIN_THREADS) {
    const bool ok = i < n;
    surv_sc[o + i] = ok ? sc[i] : -INFINITY;
    run_ix[o + i] = ok ? static_cast<int64_t>(ix[i]) + offset : -1;
  }
  if (threadIdx.x == 0) atomicAdd(status + ST_SURV, static_cast<unsigned long long>(n));
}

// Exact dense scores for small evaluation sets: grid (ceil(N/8), ceil(Q/4)), warp = one db row x 4 queries.
__global__ void scores_exact_kernel(const float* __restrict__ q, int Q, const float* __restrict__ db, int64_t N, int D,
                                    float* __restrict__ out) {
  const int64_t n = static_cast<int64_t>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  const int q0 = blockIdx.y * 4;
  const int lane = threadIdx.x & 31;
  if (n >= N) return;
  double acc[4] = {0, 0, 0, 0};
  const float4* b = reinterpret_cast<const float4*>(db + n * D);
  for (int i = lane; i < D / 4; i += 32) {
    const float4 y = __ldg(b + i);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (q0 + j < Q) {
        const float4 x = __ldg(reinterpret_cast<const float4*>(q + static_cast<int64_t>(q0 + j) * D) + i);
        acc[j] += static_cast<double>(x.x) * y.x + static_cast<double>(x.y) * y.y + static_cast<double>(x.z) * y.z +
                  static_cast<double>(x.w) * y.w;
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    double v = acc[j];
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0 && q0 + j < Q) out[static_cast<int64_t>(q0 + j) * N + n] = static_cast<float>(v);
  }
}

// alpha query expansion: out_i = normalize(q_i + sum_j db[idx_ij] * s_ij^alpha)   (test_dir.py:38-42; the mean's
// 1/(k+1) cancels in the normalisation).  partial: un-normalised neighbour sum only.
// The neighbours are taken in chunks of AQE_CHUNK weights held in shared memory; between chunks the running sums wait in
// `out` (fp32, as in the register), so every element sees the same fmaf sequence whatever the chunking.
constexpr int AQE_CHUNK = 2048;
__global__ void aqe_kernel(const float* __restrict__ q, int D, const float* __restrict__ db, const int64_t* __restrict__ nn,
                           const double* __restrict__ ns, int k, double alpha, int partial, int64_t row_offset,
                           int64_t n_rows, float* __restrict__ out) {
  extern __shared__ float wts[];  // [chunk] weights, then [chunk] local rows (as int64 pairs of floats)
  __shared__ float sh[32];
  const int kc = min(k, AQE_CHUNK);
  int64_t* rows = reinterpret_cast<int64_t*>(wts + ((kc + 1) & ~1));
  const int i = blockIdx.x;
  float ss = 0.f;
  for (int j0 = 0; j0 < k; j0 += AQE_CHUNK) {
    const int nj = min(AQE_CHUNK, k - j0);
    if (j0 > 0) __syncthreads();                     // the previous chunk's weights are no longer read
    for (int j = threadIdx.x; j < nj; j += blockDim.x) {
      int64_t r = nn[static_cast<int64_t>(i) * k + j0 + j];
      if (r >= 0 && (partial || n_rows > 0)) {       // sharded: global index -> local row of this shard, or "not mine"
                                                     // (partial sums are per shard by definition, also for an EMPTY shard)
        r -= row_offset;
        if (r < 0 || r >= n_rows) r = -1;
      }
      rows[j] = r;
      wts[j] = (r >= 0) ? static_cast<float>(pow(ns[static_cast<int64_t>(i) * k + j0 + j], alpha)) : 0.f;
    }
    __syncthreads();
    const bool last = j0 + AQE_CHUNK >= k;
    for (int c = threadIdx.x; c < D; c += blockDim.x) {
      float acc = (j0 > 0) ? out[static_cast<int64_t>(i) * D + c] : (partial ? 0.f : q[static_cast<int64_t>(i) * D + c]);
      for (int j = 0; j < nj; ++j) {
        const int64_t r = rows[j];
        if (r >= 0) acc += db[r * D + c] * wts[j];
      }
      out[static_cast<int64_t>(i) * D + c] = acc;
      if (last) ss += acc * acc;
    }
  }
  if (!partial) {
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    if (l == 0) sh[w] = ss;
    __syncthreads();
    float t = (l < (blockDim.x >> 5)) ? sh[l] : 0.f;
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    const float inv = 1.0f / sqrtf(t);
    for (int c = threadIdx.x; c < D; c += blockDim.x) out[static_cast<int64_t>(i) * D + c] *= inv;
  }
}


// ------------------------------------------------------------------------------------------------ rank counting
// AP needs, per query, only the RANKS of the labelled rows (generic.py:196-224: full argsort, junk dropped, positions
// of the positives) - not the Q x N score matrix.  For each (query, target row) the kernels below return the exact
// score s_t and above_t = the number of database rows that rank before the target under the library's order (exact
// score descending, ties -> lower index first):
//   1. exact scores of the targets                                                          (target_scores_kernel)
//   2. per query thr = min over the counted targets of s_t - eps16                          (count_thr_kernel)
//   3. wgmma filter pass: rows with fp16-path score >= thr go to the query's candidate list (PERS_EPI_SIM_FILTER);
//      every row NOT captured has exact score < s_t for every counted target
//   4. per (query, target): candidates with fp16-path score > s_t + eps16 rank before it for certain, those within
//      +-eps16 are re-scored exactly and compared (score, index)                            (rank_count_kernel)
// A query whose list overflows (a positive buried in the bulk of the score distribution) or whose band overflows is
// flagged and counted exactly from the fp32 rows instead                                    (rank_count_exact_kernel)

// one warp per target: score[t] = <q[t_q[t]], db[row - offset]> if this shard owns the row, else 0 (summed over shards)
__global__ void target_scores_kernel(const float* __restrict__ q32, const float* __restrict__ db32, int D,
                                     const int* __restrict__ t_q, const int64_t* __restrict__ t_rows, int T,
                                     int64_t offset, int64_t n_rows, double* __restrict__ t_score) {
  const int t = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (t >= T) return;
  const int64_t r = t_rows[t] - offset;
  double v = 0.0;
  if (r >= 0 && r < n_rows) v = exact_dot_warp(q32 + static_cast<int64_t>(t_q[t]) * D, db32 + r * D, D, lane);
  if (lane == 0) t_score[t] = v;
}

// thr[q] = (float, rounded down) min over counted targets of s_t - eps; +inf when the query counts nothing
__global__ void count_thr_kernel(const int* __restrict__ t_off, const unsigned char* __restrict__ t_flags,
                                 const double* __restrict__ t_score, int Q, double eps, float* __restrict__ thr) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= Q) return;
  double m = INFINITY;
  for (int t = t_off[q]; t < t_off[q + 1]; ++t)
    if (t_flags[t]) m = fmin(m, t_score[t]);
  thr[q] = (m == INFINITY) ? INFINITY : __double2float_rd(m - eps);
}

constexpr int RC_THREADS = 512;
constexpr int RC_BAND = 2048;
__global__ void __launch_bounds__(RC_THREADS) rank_count_kernel(
    const unsigned long long* __restrict__ cand, const int* __restrict__ cnt, int cap, const float* __restrict__ q32,
    const float* __restrict__ db32, int D, int64_t offset, double eps, const int* __restrict__ t_off,
    const int64_t* __restrict__ t_rows, const unsigned char* __restrict__ t_flags, const double* __restrict__ t_score,
    long long* __restrict__ above, int* __restrict__ q_over) {
  __shared__ int band[RC_BAND];
  __shared__ int s_band;
  __shared__ unsigned long long s_count;
  const int q = blockIdx.x;
  const int total = cnt[q];
  if (total > cap) {                      // uniform over the block
    if (threadIdx.x == 0) q_over[q] = 1;
    return;
  }
  const unsigned long long* c = cand + static_cast<int64_t>(q) * cap;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int t = t_off[q]; t < t_off[q + 1]; ++t) {
    if (!t_flags[t]) continue;            // uniform
    const double s = t_score[t];
    const int64_t trow = t_rows[t];
    const double hi = s + eps, lo = s - eps;
    if (threadIdx.x == 0) {
      s_band = 0;
      s_count = 0ull;
    }
    __syncthreads();
    unsigned int mine = 0;
    for (int i = threadIdx.x; i < total; i += RC_THREADS) {
      const unsigned long long e = c[i];
      const double sh = static_cast<double>(__uint_as_float(static_cast<uint32_t>(e >> 32)));
      if (sh > hi) {
        ++mine;
      } else if (sh >= lo) {
        const int pos = atomicAdd(&s_band, 1);
        if (pos < RC_BAND) band[pos] = static_cast<int>(e & 0xffffffffu);
      }
    }
    __syncthreads();
    const int nb = s_band;
    if (nb > RC_BAND) {                   // uniform: too many near-ties for the shared-memory band
      if (threadIdx.x == 0) q_over[q] = 1;
      return;
    }
    for (int w = warp; w < nb; w += RC_THREADS / 32) {
      const int row = band[w];
      const double sc = exact_dot_warp(q32 + static_cast<int64_t>(q) * D, db32 + static_cast<int64_t>(row) * D, D, lane);
      const int64_t g = static_cast<int64_t>(row) + offset;
      if (lane == 0 && g != trow && ranks_before(sc, g, s, trow)) ++mine;
    }
    for (int o = 16; o > 0; o >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, o);
    if (lane == 0 && mine) atomicAdd(&s_count, static_cast<unsigned long long>(mine));
    __syncthreads();
    if (threadIdx.x == 0) above[t] = static_cast<long long>(s_count);
    __syncthreads();
  }
}

// Exact fallback, one query per blockIdx.y: every database row is scored exactly (warp per row, fp64) and compared
// with the query's counted targets.  Reads the whole fp32 shard once per query.
constexpr int RCE_THREADS = 256;
__global__ void __launch_bounds__(RCE_THREADS) rank_count_exact_kernel(
    const float* __restrict__ q32, const float* __restrict__ db32, int D, int64_t n_rows, int64_t offset,
    const int* __restrict__ q_list, const int* __restrict__ t_off, const int64_t* __restrict__ t_rows,
    const unsigned char* __restrict__ t_flags, const double* __restrict__ t_score, unsigned long long* __restrict__ above) {
  extern __shared__ unsigned int cnts[];                   // [max targets per query of this launch]
  const int q = q_list[blockIdx.y];
  const int t0 = t_off[q], nt = t_off[q + 1] - t0;
  for (int i = threadIdx.x; i < nt; i += RCE_THREADS) cnts[i] = 0u;
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t wstride = static_cast<int64_t>(gridDim.x) * (RCE_THREADS / 32);
  for (int64_t r = static_cast<int64_t>(blockIdx.x) * (RCE_THREADS / 32) + warp; r < n_rows; r += wstride) {
    const double sc = exact_dot_warp(q32 + static_cast<int64_t>(q) * D, db32 + r * D, D, lane);
    const int64_t g = r + offset;
    for (int i = lane; i < nt; i += 32) {
      if (!t_flags[t0 + i]) continue;
      const double s = t_score[t0 + i];
      const int64_t trow = t_rows[t0 + i];
      if (g != trow && ranks_before(sc, g, s, trow)) atomicAdd(&cnts[i], 1u);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < nt; i += RCE_THREADS)
    if (cnts[i]) atomicAdd(above + t0 + i, static_cast<unsigned long long>(cnts[i]));
}


// Merge G per-shard lists that are each already ordered (score desc, index asc; empty slots = index -1 at the tail):
// the final position of an entry = its position in its own list + the number of entries of every other list that come
// before it (binary search) - no sorting network, no barriers after the load.  One block per query.
// x.world > 0: the lists are the ones the peers stored into this rank's list table (waits for their flags); the last block
// then opens the next epoch of the exchange.
__global__ void __launch_bounds__(1024) merge_lists_kernel(const double* in_score, const int64_t* in_idx,
                                                          int G, int k, int64_t shard_stride, double* __restrict__ out_score,
                                                          int64_t* __restrict__ out_idx, const PeerX x,
                                                          unsigned long long* status) {
  extern __shared__ uint8_t sm[];
  __shared__ int s_valid;
  const int q = blockIdx.x;
  const int n = G * k;
  double* sc = reinterpret_cast<double*>(sm);
  int64_t* ix = reinterpret_cast<int64_t*>(sc + n);
  if (x.world > 0) {
    const uint32_t epoch = x_epoch(x);
    if (threadIdx.x == 0) x_wait_flags(x, X_OFF_FLIST, epoch, status);
    const size_t base = static_cast<size_t>(epoch & 1u) * x.world * x_list_elems(x.max_q, x.max_k);
    in_score = reinterpret_cast<const double*>(x.peer[x.rank] + x_off_score(x.world, x.max_q)) + base;
    in_idx = reinterpret_cast<const int64_t*>(x.peer[x.rank] + x_off_idx(x.world, x.max_q, x.max_k)) + base;
    shard_stride = static_cast<int64_t>(x_list_elems(x.max_q, x.max_k));
  }
  if (threadIdx.x == 0) s_valid = 0;
  __syncthreads();                                        // (peer mode: the flags were acquired by thread 0)
  for (int e = threadIdx.x; e < n; e += blockDim.x) {
    const int64_t src = static_cast<int64_t>(e / k) * shard_stride + static_cast<int64_t>(q) * k + e % k;
    sc[e] = __ldcg(in_score + src);
    ix[e] = __ldcg(in_idx + src);
  }
  __syncthreads();
  int my_valid = 0;
  for (int e = threadIdx.x; e < n; e += blockDim.x) {
    const int g = e / k, j = e - g * k;
    const double se = sc[e];
    const int64_t ie = ix[e];
    if (ie < 0) continue;
    ++my_valid;
    int rank = j;
    for (int h = 0; h < G; ++h)
      if (h != g) rank += rank_in_run(sc + h * k, ix + h * k, k, se, ie, [](auto p) { return *p; });
    if (rank < k) {
      out_score[static_cast<int64_t>(q) * k + rank] = se;
      out_idx[static_cast<int64_t>(q) * k + rank] = ie;
    }
  }
  if (my_valid) atomicAdd(&s_valid, my_valid);
  __syncthreads();
  for (int r = s_valid + threadIdx.x; r < k; r += blockDim.x) {      // fewer than k rows in the whole database
    out_score[static_cast<int64_t>(q) * k + r] = -INFINITY;
    out_idx[static_cast<int64_t>(q) * k + r] = -1;
  }
  if (x.world > 0) {                                      // last block: this search is over, open the next epoch
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned int* cnt = reinterpret_cast<unsigned int*>(x.peer[x.rank] + X_OFF_CNT) + 2;
      if (atomicAdd(cnt, 1u) == gridDim.x - 1u) {
        *cnt = 0u;
        uint32_t* ep = reinterpret_cast<uint32_t*>(x.peer[x.rank] + X_OFF_EPOCH);
        *ep = *ep + 1u;
      }
    }
  }
}

// The same rank-based merge with the runs read from global memory, one thread per entry, for merges that do not fit in
// shared memory: run g of query q holds L entries at g * run_stride + q * q_stride, ordered (score desc, index asc), empty
// entries (index -1) only at its tail.  cnt != nullptr: query q has only ceil(min(cnt[q], cnt_cap) / L) runs.  An entry
// at position j >= k of its own run cannot reach the first k, so only the first min(L, k) entries of a run take part.
// The output must already hold (-inf, -1): every entry that ranks below k overwrites exactly one slot.
__global__ void merge_runs_kernel(const double* __restrict__ in_score, const int64_t* __restrict__ in_idx, int G, int L,
                                  int64_t run_stride, int64_t q_stride, const int* __restrict__ cnt, int cnt_cap, int Q,
                                  int k, double* __restrict__ out_score, int64_t* __restrict__ out_idx) {
  const int Lk = min(L, k);
  const int64_t e = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  for (int q = blockIdx.y; q < Q; q += gridDim.y) {
    const int Gq = cnt ? (min(cnt[q], cnt_cap) + L - 1) / L : G;
    if (e >= static_cast<int64_t>(Gq) * Lk) continue;
    const int g = static_cast<int>(e / Lk), j = static_cast<int>(e - static_cast<int64_t>(g) * Lk);
    const double* sq = in_score + static_cast<int64_t>(q) * q_stride;
    const int64_t* iq = in_idx + static_cast<int64_t>(q) * q_stride;
    const double se = __ldcg(sq + g * run_stride + j);
    const int64_t ie = __ldcg(iq + g * run_stride + j);
    if (ie < 0) continue;
    int rank = j;
    for (int h = 0; h < Gq && rank < k; ++h)
      if (h != g)
        rank += rank_in_run(sq + h * run_stride, iq + h * run_stride, Lk, se, ie, [](auto p) { return __ldcg(p); });
    if (rank < k) {
      out_score[static_cast<int64_t>(q) * k + rank] = se;
      out_idx[static_cast<int64_t>(q) * k + rank] = ie;
    }
  }
}

// ------------------------------------------------------------------------------------------------ range search / join
// Candidates of rows q0 .. q0 + nq of a block, one warp per candidate: the exact score (exact_dot_warp, row of the block
// first) and the database row, into the [nq][cap2] layout of sort_runs_merge.  Lists hold cnt[q] <= cap entries here.
__global__ void join_rescore_kernel(const unsigned long long* __restrict__ cand, const int* __restrict__ cnt, int cap,
                                    int q0, const float* __restrict__ a32, const float* __restrict__ db32, int D,
                                    int64_t col0, int cap2, int* __restrict__ rows, double* __restrict__ sc) {
  const int q = blockIdx.y;
  const int n = cnt[q0 + q];
  const int wpb = blockDim.x >> 5, lane = threadIdx.x & 31;
  const unsigned long long* c = cand + static_cast<int64_t>(q0 + q) * cap;
  const float* a = a32 + static_cast<int64_t>(q0 + q) * D;
  for (int w = blockIdx.x * wpb + (threadIdx.x >> 5); w < n; w += gridDim.x * wpb) {
    const int64_t row = col0 + static_cast<int64_t>(c[w] & 0xffffffffu);
    const double e = exact_dot_warp(a, db32 + row * D, D, lane);
    if (lane == 0) {
      rows[static_cast<int64_t>(q) * cap2 + w] = static_cast<int>(row);
      sc[static_cast<int64_t>(q) * cap2 + w] = e;
    }
  }
}

// Per row of the sub-block: the ordered list (score desc) keeps its prefix with e >= tau.
__global__ void join_kept_kernel(const double* __restrict__ out_sc, int K, const int* __restrict__ cnt, int q0, int nq,
                                 double tau, int* __restrict__ kept) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= nq) return;
  const double* s = out_sc + static_cast<int64_t>(q) * K;
  int lo = 0, hi = cnt[q0 + q];
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (s[mid] >= tau) lo = mid + 1; else hi = mid;
  }
  kept[q] = lo;
}

// The kept prefixes -> the result CSR at off[q] (offsets of this sub-block, relative to res_*).
__global__ void join_emit_kernel(const double* __restrict__ out_sc, const int64_t* __restrict__ out_ix, int K,
                                 const int* __restrict__ kept, const int64_t* __restrict__ off, int64_t index_offset,
                                 double* __restrict__ res_sc, int64_t* __restrict__ res_ix) {
  const int q = blockIdx.y;
  const int n = kept[q];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    res_sc[off[q] + i] = out_sc[static_cast<int64_t>(q) * K + i];
    res_ix[off[q] + i] = out_ix[static_cast<int64_t>(q) * K + i] + index_offset;
  }
}

}  // namespace

int sort_runs_merge(const int* rows, const int* cnt, int cap2, double* sc, int64_t* run_ix, int Q, int k,
                    int64_t row_offset, unsigned long long* status, double* out_score, int64_t* out_idx,
                    cudaStream_t stream) {
  const int runs = cap2 / SORT_RUN;
  deep_run_sort_kernel<<<dim3(runs, Q), FIN_THREADS, 0, stream>>>(rows, cnt, cap2, row_offset, sc, run_ix, status);
  const int64_t n = static_cast<int64_t>(Q) * k;
  fill_empty_result_kernel<<<static_cast<unsigned>(ceil_div(n, 256)), 256, 0, stream>>>(out_score, out_idx, n);
  const int64_t elems = static_cast<int64_t>(runs) * std::min(SORT_RUN, k);
  merge_runs_kernel<<<dim3(static_cast<unsigned>(ceil_div(elems, 256)), Q), 256, 0, stream>>>(
      sc, run_ix, runs, SORT_RUN, SORT_RUN, cap2, cnt, cap2, Q, k, out_score, out_idx);
  count_launch(3);
  DIRB_CUDA(cudaGetLastError());
  return 0;
}
}  // namespace dirb

using namespace dirb;

// Encoded 2-D tensor maps, kept per (base, rows, box): a search re-uses the same three maps every call.
struct TmapCache {
  struct E { const void* base; uint64_t inner, outer; uint32_t box; CUtensorMap m; };
  std::vector<E> es;
  int get(const void* base, uint64_t inner, uint64_t outer, uint32_t box, const CUtensorMap** out) {
    for (auto& e : es)
      if (e.base == base && e.inner == inner && e.outer == outer && e.box == box) { *out = &e.m; return 0; }
    if (es.size() >= 16) es.erase(es.begin());
    E e{base, inner, outer, box, {}};
    DIRB_TRY(encode_tmap_2d(&e.m, base, inner, outer, inner * 2, 64, box));
    es.push_back(e);
    *out = &es.back().m;
    return 0;
  }
};

// CUDA events marking the phases of a call (option "profile"), created on first use.
template <int N>
struct PhaseEvents {
  cudaEvent_t ev[N] = {};
  void mark(int i, cudaStream_t stream) {
    if (i >= N) return;
    if (!ev[i]) cudaEventCreate(&ev[i]);
    cudaEventRecord(ev[i], stream);
  }
  float ms(int i, int j) const {       // 0 when either event is missing or incomplete
    float t = 0;
    if (cudaEventElapsedTime(&t, ev[i], ev[j]) != cudaSuccess) t = 0;
    return t;
  }
  void destroy() {
    for (auto e : ev)
      if (e) cudaEventDestroy(e);
  }
};

struct dirb200_index {
  int device = 0, dim = 0;
  const float* db32 = nullptr;
  const __half* db16 = nullptr;
  int64_t N = 0, offset = 0;
  bool has_db = false;
  double eps16 = 1.2e-3;
  int64_t sample_rows = 0;
  int cand_cap = 0;          // 0 = auto
  int count_cap = 0;         // candidate capacity per query of dirb200_index_rank_count (0 = 32768)
  double count_eps = 0;      // dirb200_index_count_ge: absolute score-error bound (0 = derived from the norms per call)
  int band_cap = 0;          // dirb200_index_count_ge: band-list capacity (0 = 1 << 20 entries)
  int retries = 1;           // gated retry passes enqueued after the first filter pass (device-side predicate)
  int deferred = 0;          // 1 = search calls never synchronise; the caller collects the status (dirb200_index_check)
  double ws_budget = 4.0 * (1 << 30);   // search workspace bound in bytes: sets the largest query block (search_max_queries)
  // workspaces (grown on demand)
  void* ws = nullptr;
  size_t ws_bytes = 0;
  unsigned long long* h_status = nullptr;   // pinned copy of the device status block
  cudaEvent_t status_ev = nullptr;
  bool status_pending = false;
  int status_cap2 = 0;
  double status_band = 0;
  int64_t stats[5] = {0, 0, 0, 0, 0};
  float* sel_own = nullptr;        // selection thresholds of the single-shard entry point
  size_t sel_bytes = 0;
  // state of a search between dirb200_index_search_begin and _finish
  struct Pending {
    bool active = false;
    int Q = 0, k = 0, cap = 0, cap2 = 0, mark_i = 0;
    int64_t S = 0, launches0 = 0;
    float band = 0;
    int* cnt = nullptr;
    unsigned long long* cand = nullptr;
    unsigned long long* status = nullptr;
    float* kth_k = nullptr;
    // between the seed half and the filter half of phase 1 (the sharded search exchanges seed bounds in between)
    float* thr = nullptr;
    float* dense = nullptr;
    float* sel_dev = nullptr;
    __half* q16 = nullptr;
    int* gates = nullptr;
    int64_t S_ld = 0;
    bool small = false;
    int ks = 0;
    // deep path (k > 1024): survivors in global memory, in sort_runs_merge's layout
    SortScratch surv{};
    int* surv_cnt = nullptr;
    // filtered search: the bitmap rows of this block's queries (null = unfiltered)
    const uint32_t* allow = nullptr;
    int64_t allow_ld = 0, allow_bit0 = 0;
  } pend;
  // range search / self-join: workspace, options and the last result (CSR, kept until the next call)
  int join_cap = 0;                // candidate capacity per row of the first filter pass (0 = min(columns, 4096))
  void* jws = nullptr;             // filter pass: fp16 queries, thresholds, counts, candidate lists
  size_t jws_bytes = 0;
  void* jws2 = nullptr;            // re-scoring and sort buffers of a sub-block
  size_t jws2_bytes = 0;
  double* res_sc = nullptr;
  int64_t* res_ix = nullptr;
  size_t res_cap = 0;              // entries
  std::vector<int64_t> res_off;    // host CSR offsets of the last result
  int64_t join_stats[5] = {0, 0, 0, 0, 0};   // candidates, pairs, filter re-runs, filter launches, tiles
  double join_ms[3] = {0, 0, 0};   // option profile: filter passes, exact re-scoring, sort + compaction
  PhaseEvents<4> jev;
  int nearest_cap = 16;             // dirb200_index_nearest: most candidate groups before a row is re-scored in full
  int64_t nearest_stats[3] = {0, 0, 0};   // rows with > 1 candidate group, rows re-scored in full, centres re-scored
  // inverted lists (dirb200_index_set_lists): caller-owned fp16 rows in list order, list position -> row, K + 1 offsets
  const __half* l16 = nullptr;
  const int64_t* lperm = nullptr;
  const int64_t* lcell_off = nullptr;
  int lists_k = 0;
  void* lws[2] = {nullptr, nullptr};   // list search: [0] pair counts and offsets, [1] tile table, packed queries, lists
  size_t lws_bytes[2] = {0, 0};
  int64_t lists_stats[6] = {0, 0, 0, 0, 0, 0};   // pairs, query rows issued, tiles, probed rows, candidates, re-runs
  double lists_ms[4] = {0, 0, 0, 0};             // option profile: table build, GMAX pass + seed, FILTER pass, finish
  PhaseEvents<5> lev;
  TmapCache tmaps;
  int profile = 0;                 // option "profile": time the phases of a search with CUDA events
  PhaseEvents<10> ev;              // separate from jev / lev: the list search's finish marks these
  double phase_ms[9] = {};
  // filter of the exact search (dirb200_index_set_allow): caller-owned bitmap, words per query row (0 = shared), bit of
  // local row 0; its seed buffers live in a workspace of their own
  const uint32_t* allow = nullptr;
  int64_t allow_ld = 0, allow_bit0 = 0;
  void* aws = nullptr;
  size_t aws_bytes = 0;
};

// Similarity GEMM on the persistent wgmma kernel (conv_pers.cuh): A = queries [Q][D], B = database rows [rows][D],
// 128 x 128 tiles, K = D.  Tiles are ordered query-tile-fastest, so CTAs running at the same time share the streamed
// database tile (L2) and the database is read from HBM once.  Encoded tensor maps are kept per (base, rows) in the
// handle: a search re-uses the same three maps every call.  With a tile table (PERS_EPI_SIM_LGMAX / _LFILTER, the list
// search) the launch runs its n_tiles entries instead of the Q x rows grid, A rows being the table's query slots.
struct SimArgs {
  float* dense = nullptr; int64_t dense_ld = 0;
  const float* thr = nullptr; unsigned long long* cand = nullptr; int* cand_cnt = nullptr; int cand_cap = 0;
  const int* gate = nullptr;
  const int4* tiles = nullptr; int64_t n_tiles = 0; const int* slot_q = nullptr; const int64_t* gbase = nullptr;
  const uint32_t* allow = nullptr; int64_t allow_ld = 0, allow_bit0 = 0;
};
static int sim_gemm(dirb200_index* h, int epi, const __half* q16, int64_t Q, const __half* db16, int64_t rows, int D,
                    const SimArgs& a, cudaStream_t stream) {
  constexpr int BN = 128;
  DIRB_REQUIRE(Q < (int64_t(1) << 31), DIRB200_ENOTSUP, "too many tiles");
  const CUtensorMap* tm;
  DIRB_TRY(h->tmaps.get(q16, D, Q, 128, &tm));
  const CUtensorMap a_copy = *tm;                 // `get` may reallocate the vector: copy before the second lookup
  DIRB_TRY(h->tmaps.get(db16, D, rows, BN, &tm));
  const CUtensorMap b_copy = *tm;
  ConvPersParams p{};
  p.a_spatial = 0;
  p.taps = 1; p.kw_taps = 1; p.cin_blocks = D / 64; p.stride = 1; p.pad = 0;
  p.tw = 128; p.th = 1; p.nb = 1; p.tiles_w = 1; p.tiles_h = 1;
  p.M = static_cast<int>(Q);
  p.N = static_cast<int>(rows);
  p.n_tiles = static_cast<int>(ceil_div(rows, BN));
  p.m_tiles = static_cast<int>(ceil_div(Q, 128));
  p.m_fastest = 1;
  int64_t total = static_cast<int64_t>(p.m_tiles) * p.n_tiles;
  // the self-join launches the tiles on or above the diagonal only (decode_tile_tri)
  if (epi == PERS_EPI_SIM_JOIN) total -= static_cast<int64_t>(p.m_tiles) * (p.m_tiles - 1) / 2;
  if (a.tiles) total = a.n_tiles;
  DIRB_REQUIRE(total < (int64_t(1) << 31), DIRB200_ENOTSUP, "too many tiles");
  p.total_tiles = static_cast<int>(total);
  p.dense = a.dense; p.dense_ld = a.dense_ld;
  p.thr = a.thr; p.cand = a.cand; p.cand_cnt = a.cand_cnt; p.cand_cap = a.cand_cap;
  p.gate = a.gate;
  p.tiles = a.tiles; p.slot_q = a.slot_q; p.gbase = a.gbase;
  if (a.tiles) p.perm = h->lperm;
  p.allow = a.allow; p.allow_ld = a.allow_ld; p.allow_bit0 = a.allow_bit0;
  const int sms = num_sms();
  switch (epi) {
    case PERS_EPI_SIM_DENSE: return conv_pers_launch<BN, 6, PERS_EPI_SIM_DENSE>(a_copy, b_copy, a_copy, a_copy, p, sms, stream);
    case PERS_EPI_SIM_GMAX: return conv_pers_launch<BN, 6, PERS_EPI_SIM_GMAX>(a_copy, b_copy, a_copy, a_copy, p, sms, stream);
    case PERS_EPI_SIM_JOIN: return conv_pers_launch<BN, 6, PERS_EPI_SIM_JOIN>(a_copy, b_copy, a_copy, a_copy, p, sms, stream);
    case PERS_EPI_SIM_LGMAX: return conv_pers_launch<BN, 6, PERS_EPI_SIM_LGMAX>(a_copy, b_copy, a_copy, a_copy, p, sms, stream);
    case PERS_EPI_SIM_LFILTER:
      return conv_pers_launch<BN, 6, PERS_EPI_SIM_LFILTER>(a_copy, b_copy, a_copy, a_copy, p, sms, stream);
    case PERS_EPI_SIM_FILTER_ALLOW:
      return conv_pers_launch<BN, 6, PERS_EPI_SIM_FILTER_ALLOW>(a_copy, b_copy, a_copy, a_copy, p, sms, stream);
    default: return conv_pers_launch<BN, 6, PERS_EPI_SIM_FILTER>(a_copy, b_copy, a_copy, a_copy, p, sms, stream);
  }
}

namespace dirb {
namespace {
// ------------------------------------------------------------------------------------------------ nearest row
// dirb200_index_nearest (DESIGN.md section 4.9, rules K2 / K3), per block of queries:
//   1. queries to fp16 (nearest_prep_kernel);
//   2. one PERS_EPI_SIM_GMAX pass: G[q][g] = fp16-path maximum of the 32 rows 32g .. 32g + 31;
//   3. nearest_kernel, one block per query: M = max_g G, t = M - 2 eps16 rounded down to fp32; the groups with G >= t
//      hold every row whose exact score can be the best (its group reaches e* - eps16 >= M - 2 eps16), and are
//      re-scored exactly (exact_dot_warp); more than nearest_cap such groups -> every row is re-scored.  The best
//      (score desc, row asc) is the search's top-1.
constexpr int NEAREST_THREADS = 256;
constexpr int NEAREST_MAX_CAP = 256;

__global__ void nearest_prep_kernel(const float* __restrict__ q32, __half* __restrict__ q16, int64_t n) {
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    q16[i] = __float2half_rn(q32[i]);
}

__global__ void __launch_bounds__(NEAREST_THREADS) nearest_kernel(const float* __restrict__ G, int ng, const float* __restrict__ q32,
                                                                  const float* __restrict__ db32, int64_t K, int D,
                                                                  double eps16, int cap, int64_t offset,
                                                                  int64_t* __restrict__ labels, double* __restrict__ scores,
                                                                  unsigned long long* __restrict__ stats) {
  __shared__ float red[NEAREST_THREADS / 32];
  __shared__ int groups[NEAREST_MAX_CAP];
  __shared__ int n_groups;
  __shared__ double best_s[NEAREST_THREADS / 32];
  __shared__ int64_t best_c[NEAREST_THREADS / 32];
  const int q = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float* g = G + static_cast<int64_t>(q) * ng;
  float m = -INFINITY;
  for (int j = threadIdx.x; j < ng; j += NEAREST_THREADS) m = fmaxf(m, g[j]);
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if (lane == 0) red[warp] = m;
  if (threadIdx.x == 0) n_groups = 0;
  __syncthreads();
  m = red[0];
  for (int w = 1; w < NEAREST_THREADS / 32; ++w) m = fmaxf(m, red[w]);
  const double x = static_cast<double>(m) - 2.0 * eps16;
  float t = static_cast<float>(x);
  if (static_cast<double>(t) > x) t = nextafterf(t, -INFINITY);
  for (int j = threadIdx.x; j < ng; j += NEAREST_THREADS)
    if (g[j] >= t) {
      const int pos = atomicAdd(&n_groups, 1);
      if (pos < cap) groups[pos] = j;
    }
  __syncthreads();
  const int nc = n_groups;
  const bool full = nc > cap;
  const int64_t n_rows = full ? K : static_cast<int64_t>(nc) * 32;
  const float* a = q32 + static_cast<int64_t>(q) * D;
  double bs = -INFINITY;
  int64_t bc = INT64_MAX;
  unsigned long long scored = 0;
  for (int64_t j = warp; j < n_rows; j += NEAREST_THREADS / 32) {
    const int64_t c = full ? j : static_cast<int64_t>(groups[j >> 5]) * 32 + (j & 31);
    if (c >= K) continue;                                      // uniform over the warp
    const double e = exact_dot_warp(a, db32 + c * D, D, lane);
    if (ranks_before(e, c, bs, bc)) { bs = e; bc = c; }
    ++scored;
  }
  if (lane == 0) {
    best_s[warp] = bs;
    best_c[warp] = bc;
    atomicAdd(stats + 2, scored);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < NEAREST_THREADS / 32; ++w)
      if (ranks_before(best_s[w], best_c[w], bs, bc)) { bs = best_s[w]; bc = best_c[w]; }
    labels[q] = offset + bc;
    scores[q] = bs;
    if (nc > 1) atomicAdd(stats, 1ull);
    if (full) atomicAdd(stats + 1, 1ull);
  }
}

}  // namespace
}  // namespace dirb

// Grow one of the index's workspaces (ws, jws, jws2, lws[i]) to `need` bytes.  Cached query maps may point into the
// buffer, so they are dropped when it moves.
static int grow_ws(dirb200_index* h, void** buf, size_t* bytes, size_t need) {
  if (need > *bytes) h->tmaps.es.clear();
  return grow_device(buf, bytes, need);
}

extern "C" {

int dirb200_index_create(int device, int dim, dirb200_index** out) {
  DIRB_REQUIRE(out != nullptr, DIRB200_EINVAL, "null out");
  DIRB_TRY(dirb200_device_check(device));
  DIRB_REQUIRE(dim > 0 && dim % 64 == 0, DIRB200_ENOTSUP, "descriptor dim must be a multiple of 64 (got %d)", dim);
  auto* h = new dirb200_index();
  h->device = device;
  h->dim = dim;
  *out = h;
  return 0;
}

int dirb200_index_set_db(dirb200_index* h, const float* db32_dev, const void* db16_dev, int64_t N,
                         int64_t index_offset) {
  DIRB_REQUIRE(h && N >= 0 && (N == 0 || (db32_dev && db16_dev)), DIRB200_EINVAL, "bad db arguments");   // an empty shard has no buffers
  DIRB_REQUIRE(N < (int64_t(1) << 31) - 256, DIRB200_ENOTSUP, "shard too large (%lld rows)", (long long)N);
  h->db32 = db32_dev;
  h->db16 = static_cast<const __half*>(db16_dev);
  h->N = N;
  h->offset = index_offset;
  h->has_db = true;
  h->tmaps.es.clear();
  h->l16 = nullptr;            // lists belong to the rows they were built from: a new database detaches them
  h->lperm = nullptr;
  h->lcell_off = nullptr;
  h->lists_k = 0;
  h->allow = nullptr;          // so does the filter: its bit0 numbered the old rows
  h->allow_ld = h->allow_bit0 = 0;
  return 0;
}

int dirb200_index_set_option(dirb200_index* h, const char* key, double value) {
  DIRB_REQUIRE(h && key, DIRB200_EINVAL, "null");
  const std::string k(key);
  if (k == "eps16") h->eps16 = value;
  else if (k == "sample_rows") h->sample_rows = static_cast<int64_t>(value);
  else if (k == "cand_cap") h->cand_cap = static_cast<int>(value);
  else if (k == "profile") h->profile = value != 0;
  else if (k == "count_cap") h->count_cap = static_cast<int>(value);
  else if (k == "count_eps") h->count_eps = std::max(0.0, value);
  else if (k == "band_cap") h->band_cap = std::max(0, static_cast<int>(value));
  else if (k == "retries") h->retries = std::max(0, std::min(4, static_cast<int>(value)));
  else if (k == "deferred_check") h->deferred = value != 0;
  else if (k == "ws_budget") h->ws_budget = std::max(0.0, value);
  else if (k == "join_cap") h->join_cap = std::max(0, static_cast<int>(value));
  else if (k == "nearest_cap") h->nearest_cap = std::max(0, std::min(NEAREST_MAX_CAP, static_cast<int>(value)));
  else DIRB_REQUIRE(false, DIRB200_EKEY, "unknown index option '%s'", key);
  return 0;
}

// Collect the status of the last search (waits for it to finish): overflow errors + counters.
int dirb200_index_check(dirb200_index* h) {
  DIRB_REQUIRE(h, DIRB200_EINVAL, "null");
  if (!h->status_pending) return 0;
  DIRB_CUDA(cudaSetDevice(h->device));
  DIRB_CUDA(cudaEventSynchronize(h->status_ev));
  h->status_pending = false;
  const unsigned long long err = h->h_status[ST_ERR];
  h->stats[1] = static_cast<int64_t>(h->h_status[ST_CAND]);
  h->stats[2] = static_cast<int64_t>(h->h_status[ST_SURV]);
  h->stats[3] = static_cast<int64_t>(h->h_status[ST_RETRIES]);
  if (h->profile && h->pend.mark_i >= 2) {
    for (double& v : h->phase_ms) v = 0;
    for (int i = 0; i + 1 < h->pend.mark_i && i < 9; ++i) h->phase_ms[i] = h->ev.ms(i, i + 1);
  }
  DIRB_REQUIRE((err & 1ull) == 0, DIRB200_EOVERFLOW,
               "candidate buffer overflow not resolved after %d retry passes (raise option cand_cap)", h->retries);
  DIRB_REQUIRE((err & 4ull) == 0, DIRB200_EOVERFLOW,
               "sharded search: a peer rank did not publish its thresholds / lists in time (ranks out of step?)");
  DIRB_REQUIRE((err & 2ull) == 0, DIRB200_EOVERFLOW,
               "more than %d rows within 2*eps16=%g of the k-th score for some query (near-duplicate rows?)",
               h->status_cap2, h->status_band);
  return 0;
}

int dirb200_index_last_stats(dirb200_index* h, int64_t stats[5]) {
  DIRB_REQUIRE(h && stats, DIRB200_EINVAL, "null");
  if (h->status_pending) {                      // counters of a deferred search: wait for it, keep its error for _check
    DIRB_CUDA(cudaSetDevice(h->device));
    DIRB_CUDA(cudaEventSynchronize(h->status_ev));
    h->stats[1] = static_cast<int64_t>(h->h_status[ST_CAND]);
    h->stats[2] = static_cast<int64_t>(h->h_status[ST_SURV]);
    h->stats[3] = static_cast<int64_t>(h->h_status[ST_RETRIES]);
  }
  for (int i = 0; i < 5; ++i) stats[i] = h->stats[i];
  return 0;
}

int dirb200_index_last_profile(dirb200_index* h, double out9[9]) {
  DIRB_REQUIRE(h && out9, DIRB200_EINVAL, "null");
  for (int i = 0; i < 9; ++i) out9[i] = h->phase_ms[i];
  return 0;
}

int dirb200_index_destroy(dirb200_index* h) {
  if (!h) return 0;
  cudaSetDevice(h->device);
  h->ev.destroy();
  h->jev.destroy();
  h->lev.destroy();
  if (h->status_ev) cudaEventDestroy(h->status_ev);
  if (h->ws) cudaFree(h->ws);
  if (h->jws) cudaFree(h->jws);
  if (h->jws2) cudaFree(h->jws2);
  for (void* b : h->lws) if (b) cudaFree(b);
  if (h->aws) cudaFree(h->aws);
  if (h->res_sc) cudaFree(h->res_sc);
  if (h->res_ix) cudaFree(h->res_ix);
  if (h->sel_own) cudaFree(h->sel_own);
  if (h->h_status) cudaFreeHost(h->h_status);
  delete h;
  return 0;
}

// Phase 1: fp16 queries, seed pass, filter pass (+ device-gated retry passes), local k-th / k_shard-th candidate
// scores.  sel_dev[Q] receives the local k_shard-th best fp16-path score per query; with several shards the caller
// MIN-reduces it over the shards before phase 2 (k_shard = ceil(k / shards)); with one shard k_shard = k.
// Nothing here waits for the GPU: everything is enqueued on `stream`.
// Split in two halves: search_begin_seed (queries -> fp16, seed pass, seed bounds) and search_begin_filter (filter pass,
// candidate selection, gated retries).  seed2 != nullptr: the seed half also writes the k_shard-th seed bound of every
// query there - what a shard contributes to the MIN over the shards that tightens the filter threshold of the sharded
// search (thr_min_kernel, issued between the halves by dirb200_index_search_sharded_phase).
// Sizes of a search of depth k on this shard; none depends on Q.
constexpr int DEEP_K = 1024;        // k above this takes the deep finish (survivors in global memory)
constexpr int K_MAX = 1 << 27;      // keeps the per-query buffer sizes (2k, 8k entries) in int
struct SearchSizes {
  int64_t S = 0, S_ld = 0;
  bool small = false, gmax = false, deep = false;
  int cap = 0, cap2 = 0;
};
static SearchSizes search_sizes(const dirb200_index* h, int k) {
  SearchSizes z;
  const int64_t N = h->N;
  int64_t S = h->sample_rows > 0 ? h->sample_rows : std::max<int64_t>(8192, ceil_div(N, 16));
  S = std::min<int64_t>(std::min<int64_t>(S, 65536), N);
  S = std::max<int64_t>(S, std::min<int64_t>(N, 4 * static_cast<int64_t>(k)));
  const bool small = (N <= S);
  if (small) S = N;
  // at least k groups of 32 rows; k > 1024: 2k groups, so that the bound is the median group maximum, as with the
  // 2048 groups of the default sample at k = 1024 (with only k groups it is the smallest one: ~20 % of the rows pass)
  const int64_t groups = (k > DEEP_K ? 2 : 1) * static_cast<int64_t>(k);
  if (!small && S / 32 < groups) S = std::min<int64_t>(N, std::max<int64_t>(S, 32 * groups));
  // seed threshold from group maxima (1/32 of the dense traffic) whenever there are at least k groups; otherwise the
  // seed scores are dense (all N rows when 32 k >= N)
  z.gmax = !small && (S / 32 >= k);
  z.small = small;
  z.S = S;
  z.S_ld = ceil_div(z.gmax ? ceil_div(S, 32) : S, 128) * 128;   // dense row stride (16-byte aligned rows)
  const double expect = z.small ? (2.0 * k + 64) : (1.5 * k * static_cast<double>(N) / S);
  int cap = static_cast<int>(std::min<double>(std::max<double>(4096, 4 * expect), std::max<double>(1 << 18, 8.0 * k)));
  if (h->cand_cap > 0) cap = std::max(h->cand_cap, 2 * k);
  z.cap = (cap + 255) / 256 * 256;
  z.deep = k > DEEP_K;
  // survivors: the shallow finish sorts up to cap2 of them in shared memory; the deep one keeps 2k (at most N) in
  // global memory for sort_runs_merge
  z.cap2 = z.deep ? sort_run_cap(std::min<int64_t>(2 * static_cast<int64_t>(k), N)) : (k > 256 ? 2048 : 1024);
  return z;
}

// The search workspace of Q queries.
struct SearchWs {
  __half* q16;
  float *dense, *thr, *kth_k;
  int *cnt, *gates, *surv_cnt = nullptr;
  unsigned long long *cand, *status;
  SortScratch surv{};
  size_t total;
};
static SearchWs search_ws(void* base, const dirb200_index* h, const SearchSizes& z, int Q) {
  Carver c(base);
  SearchWs w;
  w.q16 = c.take<__half>(static_cast<size_t>(Q) * h->dim);
  w.dense = c.take<float>(static_cast<size_t>(Q) * z.S_ld);
  w.thr = c.take<float>(Q);
  w.cnt = c.take<int>(Q);
  w.cand = c.take<unsigned long long>(static_cast<size_t>(Q) * z.cap);
  w.kth_k = c.take<float>(Q);
  w.gates = c.take<int>(8);
  w.status = c.take<unsigned long long>(ST_WORDS);
  if (z.deep) {
    w.surv = take_sort_scratch(c, Q, z.cap2);
    w.surv_cnt = c.take<int>(Q);
  }
  w.total = c.used;
  return w;
}

// Largest query block whose workspace fits option ws_budget (at least 1).  Launches with a grid row per query (the
// dense compaction of the small path, the deep finish) limit it to 65535.
static int search_max_queries(const dirb200_index* h, int k) {
  if (h->N == 0) return 1 << 30;              // an empty shard has no workspace
  const SearchSizes z = search_sizes(h, k);
  int lo = 1, hi = (z.small || z.deep) ? 65535 : (1 << 30);
  while (lo < hi) {
    const int mid = lo + (hi - lo + 1) / 2;
    if (static_cast<double>(search_ws(nullptr, h, z, mid).total) <= h->ws_budget) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// The seed buffers of a filtered search of depth k (rule F2): the gathered fp16 seed rows, their row numbers, the AND of
// the block's bitmap rows over this shard's rows, and the number of seed rows found.  A workspace of its own (h->aws), so
// that the unfiltered layout and the query block of dirb200_index_search_max_queries do not change.
struct AllowWs {
  __half* seed16;
  int *rows, *n_seed;
  uint32_t* iw;
  size_t total;
};
static AllowWs allow_ws(void* base, const dirb200_index* h, int64_t S) {
  Carver c(base);
  AllowWs w;
  w.seed16 = c.take<__half>(static_cast<size_t>(S) * h->dim);
  w.rows = c.take<int>(S);
  w.n_seed = c.take<int>(1);
  w.iw = c.take<uint32_t>(static_cast<size_t>(ceil_div(h->N, 32)));
  w.total = c.used;
  return w;
}

// allow_row0: the block's first query within the rows of the attached bitmap (dirb200_index_search's query blocks).
static int search_begin_seed(dirb200_index* h, const float* q32, int Q, int k, int k_shard, float* sel_dev, cudaStream_t stream,
                             float* seed2, int64_t allow_row0 = 0) {
  DIRB_REQUIRE(h && q32 && sel_dev, DIRB200_EINVAL, "null argument");
  DIRB_REQUIRE(h->has_db, DIRB200_ESTATE, "index has no database attached");
  DIRB_REQUIRE(Q > 0 && k > 0 && k <= K_MAX, DIRB200_ENOTSUP, "need 0 < Q and 0 < k <= %d (got Q=%d k=%d)", K_MAX, Q, k);
  DIRB_REQUIRE(k_shard >= 1 && k_shard <= k, DIRB200_EINVAL, "k_shard must be in [1, k]");
  const int q_max = search_max_queries(h, k);
  DIRB_REQUIRE(Q <= q_max, DIRB200_ENOTSUP,
               "a search of depth k=%d takes at most %d queries per call within option ws_budget=%.0f bytes (got Q=%d; "
               "dirb200_index_search_max_queries)", k, q_max, h->ws_budget, Q);
  DIRB_CUDA(cudaSetDevice(h->device));
  DIRB_TRY(dirb200_index_check(h));          // an uncollected error of the previous search must not get lost
  const int64_t N = h->N;
  auto& P = h->pend;
  P = dirb200_index::Pending();
  P.active = true;
  P.Q = Q;
  P.k = k;
  P.launches0 = launches_total();
  P.cap2 = (k > 256) ? 2048 : 1024;
  P.sel_dev = sel_dev;
  if (h->allow) {
    P.allow = h->allow + allow_row0 * h->allow_ld;
    P.allow_ld = h->allow_ld;
    P.allow_bit0 = h->allow_bit0;
  }
  if (N == 0) {   // empty shard: nothing can be selected; +inf never lowers the MIN over the shards
    fill_f32_kernel<<<static_cast<unsigned>(ceil_div(Q, 256)), 256, 0, stream>>>(sel_dev, Q, INFINITY);
    count_launch();
    if (seed2) {
      fill_f32_kernel<<<static_cast<unsigned>(ceil_div(Q, 256)), 256, 0, stream>>>(seed2, Q, INFINITY);
      count_launch();
    }
    DIRB_CUDA(cudaGetLastError());
    return 0;
  }
  // ---- sizes, workspace carve-up
  const SearchSizes z = search_sizes(h, k);
  const int64_t S = z.S, S_ld = z.S_ld;
  const bool small = z.small, use_gmax = z.gmax;
  const float band = static_cast<float>(2.0 * h->eps16);
  P.S = S;
  P.cap = z.cap;
  P.cap2 = z.cap2;
  P.band = band;
  const bool filtered = P.allow != nullptr;
  if (filtered) {
    const double seed_bytes = static_cast<double>(S) * h->dim * 2;
    DIRB_REQUIRE(seed_bytes <= h->ws_budget, DIRB200_ENOTSUP,
                 "a filtered search of depth k=%d gathers %lld seed rows (%.0f bytes), more than option ws_budget=%.0f bytes",
                 k, static_cast<long long>(S), seed_bytes, h->ws_budget);
    DIRB_TRY(grow_ws(h, &h->aws, &h->aws_bytes, allow_ws(nullptr, h, S).total));
  }
  DIRB_TRY(grow_ws(h, &h->ws, &h->ws_bytes, search_ws(nullptr, h, z, Q).total));
  const SearchWs w = search_ws(h->ws, h, z, Q);
  P.cnt = w.cnt;
  P.cand = w.cand;
  P.kth_k = w.kth_k;
  P.status = w.status;
  P.surv = w.surv;
  P.surv_cnt = w.surv_cnt;
  const int D = h->dim;
  int* cnt = P.cnt;

  if (h->profile) h->ev.mark(P.mark_i++, stream);  // 0
  // ---- 1. queries to fp16, counters / gates / status cleared
  {
    const int64_t n = static_cast<int64_t>(Q) * D;
    const int64_t threads = std::max<int64_t>(ceil_div(n, 4), std::max<int64_t>(Q, 8));
    search_prep_kernel<<<static_cast<unsigned>(ceil_div(threads, 256)), 256, 0, stream>>>(q32, w.q16, n, cnt, Q, w.gates, 8, P.status);
    count_launch();
  }
  if (h->profile) h->ev.mark(P.mark_i++, stream);  // 1: convert
  // ---- 2f. filtered: seed pass over the first S rows allowed for every query of the block (rule F2)
  if (filtered) {
    const AllowWs aw = allow_ws(h->aws, h, S);
    const int64_t W = ceil_div(N, 32);
    allow_and_kernel<<<static_cast<unsigned>(ceil_div(W, 256)), 256, 0, stream>>>(P.allow, P.allow_ld, P.allow_bit0,
                                                                                 P.allow_ld == 0 ? 1 : Q, N, aw.iw);
    allow_seed_rows_kernel<<<1, ALLOW_SCAN_THREADS, 0, stream>>>(aw.iw, W, static_cast<int>(S), aw.rows, aw.n_seed);
    allow_gather_kernel<<<static_cast<unsigned>(ceil_div(S, 8)), 256, 0, stream>>>(h->db16, D, aw.rows, aw.n_seed,
                                                                                  static_cast<int>(S), aw.seed16);
    count_launch(3);
    SimArgs a;
    a.dense = w.dense;
    a.dense_ld = S_ld;
    DIRB_TRY(sim_gemm(h, use_gmax ? PERS_EPI_SIM_GMAX : PERS_EPI_SIM_DENSE, w.q16, Q, aw.seed16, S, D, a, stream));
    if (h->profile) h->ev.mark(P.mark_i++, stream);  // 2: seed gather + GEMM
    allow_kth_kernel<<<Q, SEL_THREADS, 0, stream>>>(w.dense, S_ld, static_cast<int>(S), use_gmax ? 1 : 0, aw.n_seed, k, band,
                                                    w.thr, seed2 ? k_shard : 0, seed2);
    count_launch();
    if (h->profile) h->ev.mark(P.mark_i++, stream);  // 3: k-th of the seed scores
  } else {
    SimArgs a;
    a.dense = w.dense;
    a.dense_ld = S_ld;
    DIRB_TRY(sim_gemm(h, use_gmax ? PERS_EPI_SIM_GMAX : PERS_EPI_SIM_DENSE, w.q16, Q, h->db16, S, D, a, stream));
    if (h->profile) h->ev.mark(P.mark_i++, stream);  // 2: seed GEMM
    const int n_vals = use_gmax ? static_cast<int>(ceil_div(S, 32)) : static_cast<int>(S);
    const int kk = static_cast<int>(std::min<int64_t>(k, n_vals));
    const int kk2 = seed2 ? static_cast<int>(std::min<int64_t>(k_shard, n_vals)) : 0;
    kth_dense_kernel<<<Q, SEL_THREADS, 0, stream>>>(w.dense, S_ld, n_vals, kk, band, w.thr, kk2, seed2);
    count_launch();
    if (h->profile) h->ev.mark(P.mark_i++, stream);  // 3: k-th of the seed scores
  }
  P.thr = w.thr;
  P.dense = w.dense;
  P.q16 = w.q16;
  P.gates = w.gates;
  P.S_ld = S_ld;
  P.small = small && !filtered;          // a filtered search always runs the filter as the GEMM pass (rule F3)
  P.ks = std::min<int>(k_shard, static_cast<int>(std::min<int64_t>(k, N)));
  DIRB_CUDA(cudaGetLastError());
  return 0;
}

static int search_begin_filter(dirb200_index* h, cudaStream_t stream) {
  auto& P = h->pend;
  DIRB_REQUIRE(P.active, DIRB200_ESTATE, "filter half of a search without its seed half");
  const int64_t N = h->N;
  if (N == 0) return 0;
  DIRB_CUDA(cudaSetDevice(h->device));
  const int Q = P.Q, k = P.k, D = h->dim, cap = P.cap, ks = P.ks;
  const bool small = P.small;
  const int64_t S_ld = P.S_ld;
  const float band = P.band;
  float* thr = P.thr;
  float* dense = P.dense;
  float* sel_dev = P.sel_dev;
  __half* q16 = P.q16;
  int* gates = P.gates;
  int* cnt = P.cnt;
  unsigned long long* cand = P.cand;
  // ---- 3./4. candidates + local k-th / k_shard-th candidate scores; pass r > 0 is armed by gate[r-1], which the
  //            selection of pass r-1 raises when some query overflowed its candidate list
  for (int r = 0; r <= h->retries; ++r) {
    const int* gate_in = r > 0 ? gates + (r - 1) : nullptr;
    if (small) {
      dim3 g(static_cast<unsigned>(ceil_div(N, 256)), static_cast<unsigned>(Q));
      dense_compact_kernel<<<g, 256, 0, stream>>>(dense, S_ld, static_cast<int>(N), thr, cand, cnt, cap, gate_in);
      count_launch();
    } else {
      SimArgs a;
      a.thr = thr;
      a.cand = cand;
      a.cand_cnt = cnt;
      a.cand_cap = cap;
      a.gate = gate_in;
      a.allow = P.allow;
      a.allow_ld = P.allow_ld;
      a.allow_bit0 = P.allow_bit0;
      DIRB_TRY(sim_gemm(h, P.allow ? PERS_EPI_SIM_FILTER_ALLOW : PERS_EPI_SIM_FILTER, q16, Q, h->db16, N, D, a, stream));
    }
    if (r == 0 && h->profile) h->ev.mark(P.mark_i++, stream);  // 4: filter pass
    cand_kth_kernel<<<Q, SEL_THREADS, 0, stream>>>(cand, cnt, cap, k, ks, band, P.kth_k, sel_dev, thr, N, gate_in, gates + r,
                                                   r == h->retries ? 1 : 0, P.status);
    count_launch();
    if (r == 0 && h->profile) h->ev.mark(P.mark_i++, stream);  // 5: candidate selection
  }
  if (h->profile) h->ev.mark(P.mark_i++, stream);  // 6: gated retry passes (empty launches unless a list overflowed)
  DIRB_CUDA(cudaGetLastError());
  return 0;
}

int dirb200_index_search_begin(dirb200_index* h, const float* q32, int Q, int k, int k_shard, float* sel_dev,
                               void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DIRB_TRY(search_begin_seed(h, q32, Q, k, k_shard, sel_dev, stream, nullptr));
  return search_begin_filter(h, stream);
}

// Phase 2: survivors (candidates within the band of max(sel, local k-th)), exact re-scoring, ordered output - one
// launch (search_finish_kernel) + an asynchronous copy of the status block.  Unless option deferred_check is set the
// call ends with dirb200_index_check (the only host synchronisation of a search).
// Asynchronous copy of the status block of the search in flight + the event dirb200_index_check waits for.
static int post_status_copy(dirb200_index* h, cudaStream_t stream) {
  if (!h->h_status) DIRB_CUDA(cudaMallocHost(reinterpret_cast<void**>(&h->h_status), ST_WORDS * 8));
  if (!h->status_ev) DIRB_CUDA(cudaEventCreateWithFlags(&h->status_ev, cudaEventDisableTiming));
  DIRB_CUDA(cudaMemcpyAsync(h->h_status, h->pend.status, ST_WORDS * 8, cudaMemcpyDeviceToHost, stream));
  DIRB_CUDA(cudaEventRecord(h->status_ev, stream));
  h->status_pending = true;
  return 0;
}

// collect: wait for the search and raise its errors now (dirb200_index_check); otherwise the caller collects them.
static int search_finish_impl(dirb200_index* h, const float* q32, const float* sel_dev, double* scores_dev, int64_t* idx_dev,
                              cudaStream_t stream, const PeerX& px, unsigned long long* x_status, bool collect) {
  auto& P = h->pend;
  DIRB_REQUIRE(P.active, DIRB200_ESTATE, "dirb200_index_search_finish without a matching _begin");
  DIRB_CUDA(cudaSetDevice(h->device));
  const int Q = P.Q, k = P.k, cap2 = P.cap2;
  P.active = false;
  if (h->N == 0) {
    if (px.world > 0) {   // an empty shard still publishes its (empty) lists: the peers wait for every rank's flag
      search_finish_kernel<<<Q, FIN_THREADS, static_cast<size_t>(cap2) * 12, stream>>>(nullptr, nullptr, 0, nullptr, sel_dev, 0.f, q32, nullptr,
                                                                                     h->dim, cap2, h->offset, k, nullptr, nullptr, x_status, px);
    } else {
      const int64_t n = static_cast<int64_t>(Q) * k;
      fill_empty_result_kernel<<<static_cast<unsigned>(ceil_div(n, 256)), 256, 0, stream>>>(scores_dev, idx_dev, n);
    }
    count_launch();
    DIRB_CUDA(cudaGetLastError());
    h->stats[0] = h->stats[1] = h->stats[2] = h->stats[3] = 0;
    h->stats[4] = launches_total() - P.launches0;
    return 0;
  }
  if (P.surv.rows != nullptr) {             // deep path, k > 1024 (never through peer memory: exchange windows hold k <= 1024)
    DIRB_REQUIRE(px.world == 0, DIRB200_ENOTSUP, "peer-exchange search needs k <= 1024");
    const int64_t sms = num_sms();
    DIRB_CUDA(cudaMemsetAsync(P.surv_cnt, 0, static_cast<size_t>(Q) * 4, stream));
    const unsigned gc = static_cast<unsigned>(std::max<int64_t>(1, std::min<int64_t>(ceil_div(8 * sms, Q), ceil_div(P.cap, 256))));
    deep_compact_kernel<<<dim3(gc, Q), 256, 0, stream>>>(P.cand, P.cnt, P.cap, P.kth_k, sel_dev, P.band, P.surv.rows, P.surv_cnt,
                                                         cap2, P.status);
    count_launch();
    if (h->profile) h->ev.mark(P.mark_i++, stream);  // 7: survivor compaction
    const unsigned gr = static_cast<unsigned>(std::max<int64_t>(1, std::min<int64_t>(ceil_div(32 * sms, Q), ceil_div(cap2, 8))));
    deep_rescore_kernel<<<dim3(gr, Q), 256, 0, stream>>>(q32, h->db32, h->dim, P.surv.rows, P.surv_cnt, cap2, P.surv.sc);
    count_launch();
    if (h->profile) h->ev.mark(P.mark_i++, stream);  // 8: exact re-scoring
    DIRB_TRY(sort_runs_merge(P.surv.rows, P.surv_cnt, cap2, P.surv.sc, P.surv.run_ix, Q, k, h->offset, P.status, scores_dev,
                             idx_dev, stream));
    if (h->profile) h->ev.mark(P.mark_i++, stream);  // 9: run sort + merge
  } else {
    const size_t smem = static_cast<size_t>(cap2) * 12;
    search_finish_kernel<<<Q, FIN_THREADS, smem, stream>>>(P.cand, P.cnt, P.cap, P.kth_k, sel_dev, P.band, q32, h->db32, h->dim,
                                                           cap2, h->offset, k, scores_dev, idx_dev, P.status, px);
    count_launch();
    DIRB_CUDA(cudaGetLastError());
    if (h->profile) h->ev.mark(P.mark_i++, stream);  // 7: survivors + exact re-scoring + sort
  }
  h->status_cap2 = cap2;
  h->status_band = P.band;
  h->stats[0] = P.S;
  h->stats[4] = launches_total() - P.launches0;
  if (px.world > 0) return 0;               // sharded search over peer memory: the merge (phase 3) can still raise error bits
  DIRB_TRY(post_status_copy(h, stream));
  return collect ? dirb200_index_check(h) : 0;
}

int dirb200_index_search_finish(dirb200_index* h, const float* q32, const float* sel_dev, double* scores_dev,
                                int64_t* idx_dev, void* stream_) {
  DIRB_REQUIRE(h && q32 && sel_dev && scores_dev && idx_dev, DIRB200_EINVAL, "null argument");
  return search_finish_impl(h, q32, sel_dev, scores_dev, idx_dev, static_cast<cudaStream_t>(stream_), PeerX{}, nullptr,
                            !h->deferred);
}

int dirb200_index_search_max_queries(dirb200_index* h, int k, int* q_max) {
  DIRB_REQUIRE(h && q_max, DIRB200_EINVAL, "null argument");
  DIRB_REQUIRE(h->has_db, DIRB200_ESTATE, "index has no database attached");
  DIRB_REQUIRE(k > 0 && k <= K_MAX, DIRB200_ENOTSUP, "need 0 < k <= %d (got k=%d)", K_MAX, k);
  *q_max = search_max_queries(h, k);
  return 0;
}

// Single-shard search = phase 1 with k_shard = k followed directly by phase 2, in blocks of at most
// dirb200_index_search_max_queries queries (one block unless Q * k outgrows option ws_budget).
int dirb200_index_search(dirb200_index* h, const float* q32, int Q, int k, double* scores_dev, int64_t* idx_dev,
                         void* stream_) {
  DIRB_REQUIRE(h && q32 && scores_dev && idx_dev, DIRB200_EINVAL, "null argument");
  DIRB_REQUIRE(Q > 0, DIRB200_ENOTSUP, "need Q > 0");
  int qb = Q;
  if (h->has_db && k > 0 && k <= K_MAX) qb = std::min(Q, search_max_queries(h, k));   // (bad arguments: _begin reports them)
  DIRB_TRY(grow_device(reinterpret_cast<void**>(&h->sel_own), &h->sel_bytes, static_cast<size_t>(qb) * 4));
  for (int q0 = 0; q0 < Q; q0 += qb) {
    const int nb = std::min(qb, Q - q0);
    const float* qq = q32 + static_cast<int64_t>(q0) * h->dim;
    const int64_t o = static_cast<int64_t>(q0) * k;
    DIRB_TRY(search_begin_seed(h, qq, nb, k, k, h->sel_own, static_cast<cudaStream_t>(stream_), nullptr, q0));
    DIRB_TRY(search_begin_filter(h, static_cast<cudaStream_t>(stream_)));
    DIRB_TRY(dirb200_index_search_finish(h, qq, h->sel_own, scores_dev + o, idx_dev + o, stream_));
  }
  return 0;
}

int dirb200_index_set_allow(dirb200_index* h, const uint32_t* words_dev, int64_t ld_words, int64_t bit0) {
  DIRB_REQUIRE(h, DIRB200_EINVAL, "null");
  h->allow = nullptr;
  h->allow_ld = h->allow_bit0 = 0;
  if (words_dev == nullptr) return 0;
  DIRB_REQUIRE(ld_words >= 0 && bit0 >= 0, DIRB200_EINVAL, "need ld_words >= 0 and bit0 >= 0");
  DIRB_REQUIRE(ld_words == 0 || ld_words * 32 >= bit0 + h->N, DIRB200_EINVAL,
               "a bitmap row of %lld words does not reach bit %lld (bit0 + N - 1)", static_cast<long long>(ld_words),
               static_cast<long long>(bit0 + h->N - 1));
  h->allow = words_dev;
  h->allow_ld = ld_words;
  h->allow_bit0 = bit0;
  return 0;
}

int dirb200_allow_exclude(uint32_t* words_dev, int Q, int64_t ld_words, const int64_t* off_dev, const int64_t* rows_dev,
                          void* stream_) {
  DIRB_REQUIRE(Q >= 0 && ld_words >= 1, DIRB200_EINVAL, "need Q >= 0 and ld_words >= 1");
  if (Q == 0) return 0;
  DIRB_REQUIRE(words_dev && off_dev && rows_dev, DIRB200_EINVAL, "null argument");
  allow_exclude_kernel<<<Q, 256, 0, static_cast<cudaStream_t>(stream_)>>>(words_dev, ld_words, off_dev, rows_dev);
  count_launch();
  DIRB_CUDA(cudaGetLastError());
  return 0;
}

// Entry points that rank, count or select rows without the filter refuse to run while one is attached.
static int no_filter(const dirb200_index* h) {
  DIRB_REQUIRE(h->allow == nullptr, DIRB200_ESTATE,
               "a filter is attached (dirb200_index_set_allow): only the top-k search applies it; detach it first");
  return 0;
}

// ---- rank counting (see the kernels above): exact scores of the labelled rows + number of rows ranking before them
int dirb200_index_target_scores(dirb200_index* h, const float* q32, int Q, const int* t_q_dev, const int64_t* t_rows_dev,
                                int T, double* t_score_dev, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DIRB_REQUIRE(h && q32 && Q > 0 && T >= 0, DIRB200_EINVAL, "bad arguments");
  DIRB_REQUIRE(h->has_db, DIRB200_ESTATE, "index has no database attached");
  DIRB_TRY(no_filter(h));
  if (T == 0) return 0;
  DIRB_REQUIRE(t_q_dev && t_rows_dev && t_score_dev, DIRB200_EINVAL, "null argument");
  DIRB_CUDA(cudaSetDevice(h->device));
  target_scores_kernel<<<static_cast<unsigned>(ceil_div(T, 8)), 256, 0, stream>>>(q32, h->db32, h->dim, t_q_dev, t_rows_dev, T,
                                                                                  h->offset, h->N, t_score_dev);
  count_launch();
  DIRB_CUDA(cudaGetLastError());
  return 0;
}

int dirb200_index_rank_count(dirb200_index* h, const float* q32, int Q, const int* t_off_host, const int* t_off_dev,
                             const int64_t* t_rows_dev, const unsigned char* t_flags_dev, const double* t_score_dev,
                             int T, int64_t* above_dev, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DIRB_REQUIRE(h && q32 && Q > 0 && T >= 0 && t_off_host, DIRB200_EINVAL, "bad arguments");
  DIRB_REQUIRE(h->has_db, DIRB200_ESTATE, "index has no database attached");
  DIRB_TRY(no_filter(h));
  if (T == 0) return 0;
  DIRB_REQUIRE(t_off_dev && t_rows_dev && t_flags_dev && t_score_dev && above_dev, DIRB200_EINVAL, "null argument");
  DIRB_REQUIRE(t_off_host[0] == 0 && t_off_host[Q] == T, DIRB200_EINVAL, "target offsets must run from 0 to T");
  DIRB_CUDA(cudaSetDevice(h->device));
  DIRB_TRY(dirb200_index_check(h));
  h->pend.active = false;                        // shares the search workspace
  const int64_t launches0 = launches_total();
  DIRB_CUDA(cudaMemsetAsync(above_dev, 0, static_cast<size_t>(T) * 8, stream));
  h->stats[0] = h->stats[1] = h->stats[2] = h->stats[3] = 0;
  if (h->N == 0) {
    h->stats[4] = launches_total() - launches0;
    return 0;
  }
  const int D = h->dim;
  const int64_t N = h->N;
  int cap = h->count_cap > 0 ? h->count_cap : 32768;
  cap = std::max(1024, (cap + 255) / 256 * 256);
  __half* q16;
  float* thr;
  int *cnt, *gates, *q_over, *q_list;
  unsigned long long *cand, *status;
  auto layout = [&](void* base) {
    Carver c(base);
    q16 = c.take<__half>(static_cast<size_t>(Q) * D);
    thr = c.take<float>(Q);
    cnt = c.take<int>(Q);
    cand = c.take<unsigned long long>(static_cast<size_t>(Q) * cap);
    gates = c.take<int>(8);
    status = c.take<unsigned long long>(ST_WORDS);
    q_over = c.take<int>(Q);
    q_list = c.take<int>(Q);
    return c.used;
  };
  DIRB_TRY(grow_ws(h, &h->ws, &h->ws_bytes, layout(nullptr)));
  layout(h->ws);
  {
    const int64_t n = static_cast<int64_t>(Q) * D;
    const int64_t threads = std::max<int64_t>(ceil_div(n, 4), std::max<int64_t>(Q, 8));
    search_prep_kernel<<<static_cast<unsigned>(ceil_div(threads, 256)), 256, 0, stream>>>(q32, q16, n, cnt, Q, gates, 8, status);
    count_launch();
  }
  DIRB_CUDA(cudaMemsetAsync(q_over, 0, static_cast<size_t>(Q) * 4, stream));
  count_thr_kernel<<<static_cast<unsigned>(ceil_div(Q, 128)), 128, 0, stream>>>(t_off_dev, t_flags_dev, t_score_dev, Q, h->eps16, thr);
  count_launch();
  {
    SimArgs a;
    a.thr = thr;
    a.cand = cand;
    a.cand_cnt = cnt;
    a.cand_cap = cap;
    DIRB_TRY(sim_gemm(h, PERS_EPI_SIM_FILTER, q16, Q, h->db16, N, D, a, stream));
  }
  rank_count_kernel<<<Q, RC_THREADS, 0, stream>>>(cand, cnt, cap, q32, h->db32, D, h->offset, h->eps16, t_off_dev, t_rows_dev,
                                                  t_flags_dev, t_score_dev, reinterpret_cast<long long*>(above_dev), q_over);
  count_launch();
  DIRB_CUDA(cudaGetLastError());
  std::vector<int> over(Q), hcnt(Q);
  DIRB_CUDA(cudaMemcpyAsync(over.data(), q_over, static_cast<size_t>(Q) * 4, cudaMemcpyDeviceToHost, stream));
  DIRB_CUDA(cudaMemcpyAsync(hcnt.data(), cnt, static_cast<size_t>(Q) * 4, cudaMemcpyDeviceToHost, stream));
  DIRB_CUDA(cudaStreamSynchronize(stream));
  std::vector<int> list;
  int max_nt = 0;
  int64_t cand_total = 0;
  for (int q = 0; q < Q; ++q) {
    cand_total += std::min(hcnt[q], cap);
    if (!over[q]) continue;
    list.push_back(q);
    max_nt = std::max(max_nt, t_off_host[q + 1] - t_off_host[q]);
    // a band overflow may have left partial counts behind
    DIRB_CUDA(cudaMemsetAsync(above_dev + t_off_host[q], 0, static_cast<size_t>(t_off_host[q + 1] - t_off_host[q]) * 8, stream));
  }
  if (!list.empty()) {
    DIRB_REQUIRE(static_cast<size_t>(max_nt) * 4 <= 200 * 1024, DIRB200_ENOTSUP, "more than 51200 labelled rows for one query");
    DIRB_CUDA(cudaMemcpyAsync(q_list, list.data(), list.size() * 4, cudaMemcpyHostToDevice, stream));
    const size_t smem = static_cast<size_t>(std::max(max_nt, 1)) * 4;
    DIRB_CUDA(cudaFuncSetAttribute(rank_count_exact_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    const int gx = static_cast<int>(std::min<int64_t>(ceil_div(N, RCE_THREADS / 32), 4 * static_cast<int64_t>(num_sms())));
    // a few queries per launch: each grid row re-reads the whole fp32 shard
    for (size_t i0 = 0; i0 < list.size(); i0 += 4096) {
      const unsigned ny = static_cast<unsigned>(std::min<size_t>(4096, list.size() - i0));
      rank_count_exact_kernel<<<dim3(gx, ny), RCE_THREADS, smem, stream>>>(
          q32, h->db32, D, N, h->offset, q_list + i0, t_off_dev, t_rows_dev, t_flags_dev, t_score_dev,
          reinterpret_cast<unsigned long long*>(above_dev));
      count_launch();
    }
    DIRB_CUDA(cudaGetLastError());
    DIRB_CUDA(cudaStreamSynchronize(stream));    // `list` is read by the async copy above
  }
  h->stats[1] = cand_total;
  h->stats[3] = static_cast<int64_t>(list.size());
  h->stats[4] = launches_total() - launches0;
  return 0;
}

// ---- threshold counts for label-based AP (kernels: label_count.cu)
int dirb200_index_count_ge(dirb200_index* h, const float* q32, int Q, const int* thr_off_dev, const float* thr_dev, int T,
                           const int64_t* skip_row_dev, int64_t* count_dev, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DIRB_REQUIRE(h && Q >= 0 && T >= 0, DIRB200_EINVAL, "bad arguments");
  DIRB_REQUIRE(h->has_db, DIRB200_ESTATE, "index has no database attached");
  DIRB_TRY(no_filter(h));
  DIRB_REQUIRE(Q <= 65535 * 64, DIRB200_ENOTSUP, "count_ge takes at most %d queries per call (got %d)", 65535 * 64, Q);
  h->stats[0] = h->stats[1] = h->stats[2] = h->stats[3] = h->stats[4] = 0;
  if (Q == 0 || T == 0) return 0;
  DIRB_REQUIRE(q32 && thr_off_dev && thr_dev && count_dev, DIRB200_EINVAL, "null argument");
  DIRB_CUDA(cudaSetDevice(h->device));
  DIRB_TRY(dirb200_index_check(h));
  h->pend.active = false;                        // shares the search workspace
  const int64_t launches0 = launches_total();
  const int cap = h->band_cap > 0 ? h->band_cap : (1 << 20);
  DIRB_TRY(grow_ws(h, &h->ws, &h->ws_bytes, count_ge_ws_bytes(Q, T, cap)));
  CountGeArgs a;
  a.q32 = q32; a.Q = Q;
  a.db32 = h->db32; a.N = h->N; a.offset = h->offset; a.D = h->dim;
  a.thr_off = thr_off_dev; a.thr = thr_dev; a.T = T;
  a.skip_row = skip_row_dev; a.count = count_dev;
  a.eps = h->count_eps; a.band_cap = cap;
  CountGeStats st;
  DIRB_TRY(count_ge_run(a, h->ws, &st, stream));
  h->stats[1] = st.band;
  h->stats[3] = st.fallback;
  h->stats[4] = launches_total() - launches0;
  return 0;
}

// ---- range search and self-join (DESIGN.md section 4.8, rules J1-J6)
// One block of rows (queries, or database rows i0 .. i0 + M of a self-join) against the database rows col0 .. N:
//   1. filter pass: the fp16 tensor-core GEMM keeps every column with fp16-path score >= thr (PERS_EPI_SIM_FILTER, or
//      PERS_EPI_SIM_JOIN over the tiles on or above the diagonal with col > row); its atomicAdd counts every match
//      exactly, also past the list capacity.  The counts come back to the host (the one synchronisation of a block); a
//      list that overflowed re-runs the block with capacity = its count, or the block is halved when that does not fit
//      option ws_budget.
//   2. exact re-scoring of the candidates (exact_dot_warp) and their order (score desc, row asc, sort_runs_merge), in
//      sub-blocks of rows whose sort buffers fit the budget; the rows with e >= tau are a prefix of each ordered list.
//   3. the prefixes are appended to the result CSR (second synchronisation, for their lengths).
// thr = tau - eps16 rounded down to fp32: every row with e >= tau has fp16-path score >= thr (rule J5).
namespace {

float join_threshold(double tau, double eps16) {
  const double x = tau - eps16;
  float f = static_cast<float>(x);
  if (static_cast<double>(f) > x) f = nextafterf(f, -INFINITY);
  return f;
}

struct JoinRun {
  dirb200_index* h;
  const float* a32;        // rows of the block side (queries, or the database itself)
  bool tri;                // self-join: the block's rows are database rows, columns start at the block's first row
  double tau;
  float thr;
  cudaStream_t stream;
};

// Filter pass of M rows (jws): their fp16 copy (none in a self-join, whose rows are the database's), thresholds, counts,
// candidate lists and status.
struct JoinFilterWs {
  __half* a16;
  float* thr;
  int* cnt;
  unsigned long long *cand, *status;
  size_t total;
};
JoinFilterWs join_filter_ws(void* base, int M, int D, int cap, bool tri) {
  Carver c(base);
  JoinFilterWs w;
  w.a16 = tri ? nullptr : c.take<__half>(static_cast<size_t>(M) * D);
  w.thr = c.take<float>(M);
  w.cnt = c.take<int>(M);
  w.cand = c.take<unsigned long long>(static_cast<size_t>(M) * cap);
  w.status = c.take<unsigned long long>(ST_WORDS);
  w.total = c.used;
  return w;
}
// Re-scoring and sort buffers of nq rows of at most K candidates (jws2): the sorted top-K of each and its kept prefix.
struct JoinSortWs {
  SortScratch s;
  double* out_sc;
  int64_t* out_ix;
  int* kept;
  int64_t* off;
  size_t total;
};
JoinSortWs join_sort_ws(void* base, int nq, int K) {
  Carver c(base);
  JoinSortWs w;
  const size_t nk = static_cast<size_t>(nq) * std::max(K, 1);
  w.s = take_sort_scratch(c, nq, sort_run_cap(std::max(K, 1)));
  w.out_sc = c.take<double>(nk);
  w.out_ix = c.take<int64_t>(nk);
  w.kept = c.take<int>(nq);
  w.off = c.take<int64_t>(nq);
  w.total = c.used;
  return w;
}

// Appends n more result entries, keeping the ones already there.
int join_reserve(dirb200_index* h, int64_t used, int64_t add, cudaStream_t stream) {
  const size_t need = static_cast<size_t>(used + add);
  if (need <= h->res_cap) return 0;
  const size_t cap = std::max(need, h->res_cap + h->res_cap / 2);
  double* sc = nullptr;
  int64_t* ix = nullptr;
  DIRB_CUDA(cudaMalloc(reinterpret_cast<void**>(&sc), cap * 8));
  DIRB_CUDA(cudaMalloc(reinterpret_cast<void**>(&ix), cap * 8));
  if (used > 0) {
    DIRB_CUDA(cudaMemcpyAsync(sc, h->res_sc, used * 8, cudaMemcpyDeviceToDevice, stream));
    DIRB_CUDA(cudaMemcpyAsync(ix, h->res_ix, used * 8, cudaMemcpyDeviceToDevice, stream));
    DIRB_CUDA(cudaStreamSynchronize(stream));
  }
  if (h->res_sc) DIRB_CUDA(cudaFree(h->res_sc));
  if (h->res_ix) DIRB_CUDA(cudaFree(h->res_ix));
  h->res_sc = sc;
  h->res_ix = ix;
  h->res_cap = cap;
  return 0;
}

// Rows r0 .. r0 + M of the block side against columns col0 .. N; appends their lists to the result.
int join_rows(const JoinRun& R, int64_t r0, int M, int64_t col0, int cap) {
  dirb200_index* h = R.h;
  const int D = h->dim;
  const int64_t ncols = h->N - col0;
  cudaStream_t stream = R.stream;
  const float* a32 = R.a32 + r0 * D;
  const auto budget = static_cast<size_t>(h->ws_budget);
  // ---- 1. filter pass (+ one re-run at the exact capacity when a list overflowed)
  std::vector<int> cnt_h(M);
  int* cnt = nullptr;
  unsigned long long* cand = nullptr;
  unsigned long long* status = nullptr;
  size_t used = 0;
  for (int pass = 0;; ++pass) {
    used = join_filter_ws(nullptr, M, D, cap, R.tri).total;
    DIRB_TRY(grow_ws(h, &h->jws, &h->jws_bytes, used));
    const JoinFilterWs f = join_filter_ws(h->jws, M, D, cap, R.tri);
    __half* a16 = R.tri ? const_cast<__half*>(h->db16) + r0 * D : f.a16;
    cnt = f.cnt;
    cand = f.cand;
    status = f.status;
    if (h->profile) h->jev.mark(0, stream);
    if (R.tri) {
      DIRB_CUDA(cudaMemsetAsync(cnt, 0, static_cast<size_t>(M) * 4, stream));
    } else {
      const int64_t n = static_cast<int64_t>(M) * D;
      const int64_t threads = std::max<int64_t>(ceil_div(n, 4), std::max<int64_t>(M, 8));
      search_prep_kernel<<<static_cast<unsigned>(ceil_div(threads, 256)), 256, 0, stream>>>(a32, a16, n, cnt, M, nullptr, 0, status);
      count_launch();
    }
    fill_f32_kernel<<<static_cast<unsigned>(ceil_div(M, 256)), 256, 0, stream>>>(f.thr, M, R.thr);
    count_launch();
    SimArgs a;
    a.thr = f.thr;
    a.cand = cand;
    a.cand_cnt = cnt;
    a.cand_cap = cap;
    DIRB_TRY(sim_gemm(h, R.tri ? PERS_EPI_SIM_JOIN : PERS_EPI_SIM_FILTER, a16, M, h->db16 + col0 * D, ncols, D, a, stream));
    const int64_t mt = ceil_div(M, 128), nt = ceil_div(ncols, 128);
    h->join_stats[3] += 1;
    h->join_stats[4] += R.tri ? mt * nt - mt * (mt - 1) / 2 : mt * nt;
    if (h->profile) h->jev.mark(1, stream);
    DIRB_CUDA(cudaMemcpyAsync(cnt_h.data(), cnt, static_cast<size_t>(M) * 4, cudaMemcpyDeviceToHost, stream));
    DIRB_CUDA(cudaStreamSynchronize(stream));
    if (h->profile) h->join_ms[0] += h->jev.ms(0, 1);
    const int cmax = *std::max_element(cnt_h.begin(), cnt_h.end());
    if (cmax <= cap) break;
    // overflow: the counts are exact, so one re-run at capacity cmax captures every candidate (rule J6)
    DIRB_REQUIRE(pass == 0, DIRB200_EOVERFLOW, "candidate count changed between two filter passes");
    const int cap_new = static_cast<int>(std::min<int64_t>(ceil_div(cmax, 256) * 256, ncols));
    const size_t sort1 = join_sort_ws(nullptr, 1, cmax).total;
    if (join_filter_ws(nullptr, M, D, cap_new, R.tri).total + sort1 <= budget) {
      cap = cap_new;
      h->join_stats[2] += 1;
      continue;
    }
    const int step = R.tri ? 128 : 1;           // a self-join block starts at a tile boundary
    DIRB_REQUIRE(M > step, DIRB200_EOVERFLOW,
                 "row %lld has %d candidates within eps16 of tau: %zu bytes of workspace needed, option ws_budget is %.0f",
                 static_cast<long long>(r0), cmax, join_filter_ws(nullptr, 1, D, cap_new, R.tri).total + sort1,
                 h->ws_budget);
    const int half = static_cast<int>(ceil_div(ceil_div(M, step), 2) * step);
    h->join_stats[2] += 1;
    DIRB_TRY(join_rows(R, r0, half, col0, cap));
    return join_rows(R, r0 + half, M - half, R.tri ? col0 + half : col0, cap);
  }
  for (int q = 0; q < M; ++q) h->join_stats[0] += cnt_h[q];
  // ---- 2./3. exact re-scoring, order, kept prefixes -> result, in sub-blocks of rows that fit the budget
  const size_t sort_budget = budget > used ? budget - used : 0;
  for (int q0 = 0; q0 < M;) {
    int nq = 0, K = 0;
    while (q0 + nq < M && nq < 65535) {
      const int K2 = std::max(K, cnt_h[q0 + nq]);
      if (nq > 0 && join_sort_ws(nullptr, nq + 1, K2).total > sort_budget) break;
      K = K2;
      ++nq;
    }
    DIRB_REQUIRE(join_sort_ws(nullptr, nq, K).total <= sort_budget || nq > 1, DIRB200_EOVERFLOW,
                 "row %lld has %d candidates within eps16 of tau: %zu bytes of workspace needed, option ws_budget is %.0f",
                 static_cast<long long>(r0 + q0), K, used + join_sort_ws(nullptr, 1, K).total, h->ws_budget);
    const int64_t base = h->res_off.back();
    if (K == 0) {
      for (int q = 0; q < nq; ++q) h->res_off.push_back(base);
      q0 += nq;
      continue;
    }
    const int cap2 = sort_run_cap(K);
    DIRB_TRY(grow_ws(h, &h->jws2, &h->jws2_bytes, join_sort_ws(nullptr, nq, K).total));
    const JoinSortWs w = join_sort_ws(h->jws2, nq, K);
    if (h->profile) h->jev.mark(1, stream);
    const int64_t sms = num_sms();
    const unsigned gr = static_cast<unsigned>(std::max<int64_t>(1, std::min<int64_t>(ceil_div(32 * sms, nq), ceil_div(K, 8))));
    join_rescore_kernel<<<dim3(gr, nq), 256, 0, stream>>>(cand, cnt, cap, q0, a32, h->db32, D, col0, cap2, w.s.rows,
                                                          w.s.sc);
    count_launch();
    if (h->profile) h->jev.mark(2, stream);
    DIRB_TRY(sort_runs_merge(w.s.rows, cnt + q0, cap2, w.s.sc, w.s.run_ix, nq, K, 0, status, w.out_sc, w.out_ix, stream));
    join_kept_kernel<<<static_cast<unsigned>(ceil_div(nq, 256)), 256, 0, stream>>>(w.out_sc, K, cnt, q0, nq, R.tau, w.kept);
    count_launch();
    std::vector<int> kept_h(nq);
    DIRB_CUDA(cudaMemcpyAsync(kept_h.data(), w.kept, static_cast<size_t>(nq) * 4, cudaMemcpyDeviceToHost, stream));
    DIRB_CUDA(cudaStreamSynchronize(stream));
    std::vector<int64_t> off_h(nq);
    int64_t t = base;
    int kmax = 0;
    for (int q = 0; q < nq; ++q) {
      off_h[q] = t - base;
      t += kept_h[q];
      kmax = std::max(kmax, kept_h[q]);
      h->res_off.push_back(t);
    }
    if (t > base) {
      DIRB_TRY(join_reserve(h, base, t - base, stream));
      DIRB_CUDA(cudaMemcpyAsync(w.off, off_h.data(), static_cast<size_t>(nq) * 8, cudaMemcpyHostToDevice, stream));
      const unsigned ge = static_cast<unsigned>(std::min<int64_t>(ceil_div(kmax, 256), 64));
      join_emit_kernel<<<dim3(ge, nq), 256, 0, stream>>>(w.out_sc, w.out_ix, K, w.kept, w.off, h->offset, h->res_sc + base,
                                                          h->res_ix + base);
      count_launch();
    }
    if (h->profile) h->jev.mark(3, stream);
    DIRB_CUDA(cudaStreamSynchronize(stream));    // off_h / kept_h leave scope; the timing events are complete
    if (h->profile) {
      h->join_ms[1] += h->jev.ms(1, 2);
      h->join_ms[2] += h->jev.ms(2, 3);
    }
    DIRB_CUDA(cudaGetLastError());
    q0 += nq;
  }
  return 0;
}

int join_begin(dirb200_index* h, double tau) {
  DIRB_REQUIRE(h->has_db, DIRB200_ESTATE, "index has no database attached");
  DIRB_TRY(no_filter(h));
  DIRB_REQUIRE(std::isfinite(tau), DIRB200_EINVAL, "tau must be finite");
  DIRB_CUDA(cudaSetDevice(h->device));
  DIRB_TRY(dirb200_index_check(h));
  h->res_off.assign(1, 0);
  for (auto& v : h->join_stats) v = 0;
  for (auto& v : h->join_ms) v = 0;
  return 0;
}

// Largest block of rows whose first filter pass fits half of option ws_budget (the rest is for the sort buffers), and
// whose fp16 rows stay resident in L2 (16 MiB): in the m-fastest tile order every column tile meets all of the block's
// row tiles, so a larger block re-reads its rows from HBM for each column tile and the GEMM becomes bandwidth-bound.
int join_block_rows(const dirb200_index* h, int cap, bool tri) {
  const int step = tri ? 128 : 1;
  const int l2_rows = std::max(step, (16 << 20) / (2 * h->dim) / 128 * 128);
  int lo = step, hi = std::min(65535 / step * step, l2_rows);
  while (lo < hi) {
    const int mid = (lo + hi + step) / 2 / step * step;
    if (static_cast<double>(join_filter_ws(nullptr, mid, h->dim, cap, tri).total) <= 0.5 * h->ws_budget) lo = mid;
    else hi = mid - step;
  }
  return lo;
}

int join_first_cap(const dirb200_index* h, int64_t ncols) {
  if (h->join_cap > 0) return h->join_cap;
  return static_cast<int>(std::max<int64_t>(1, std::min<int64_t>(ncols, 4096)));
}

}  // namespace

int dirb200_index_range_search(dirb200_index* h, const float* q32, int Q, double tau, int64_t* total_out, void* stream_) {
  DIRB_REQUIRE(h && q32 && total_out && Q > 0, DIRB200_EINVAL, "bad arguments");
  DIRB_TRY(join_begin(h, tau));
  const JoinRun R{h, q32, false, tau, join_threshold(tau, h->eps16), static_cast<cudaStream_t>(stream_)};
  if (h->N > 0) {
    const int cap = join_first_cap(h, h->N);
    const int qb = join_block_rows(h, cap, false);
    for (int q0 = 0; q0 < Q; q0 += qb) DIRB_TRY(join_rows(R, q0, std::min(qb, Q - q0), 0, cap));
  } else {
    h->res_off.assign(static_cast<size_t>(Q) + 1, 0);
  }
  h->join_stats[1] = h->res_off.back();
  *total_out = h->res_off.back();
  return 0;
}

int dirb200_index_self_join(dirb200_index* h, int64_t row0, int64_t row1, double tau, int64_t* total_out, void* stream_) {
  DIRB_REQUIRE(h && total_out, DIRB200_EINVAL, "bad arguments");
  DIRB_TRY(join_begin(h, tau));
  DIRB_REQUIRE(row0 >= 0 && row0 <= row1 && row1 <= h->N && row0 % 128 == 0, DIRB200_EINVAL,
               "need 0 <= row0 <= row1 <= N with row0 a multiple of 128 (got %lld, %lld, N = %lld)",
               static_cast<long long>(row0), static_cast<long long>(row1), static_cast<long long>(h->N));
  const JoinRun R{h, h->db32, true, tau, join_threshold(tau, h->eps16), static_cast<cudaStream_t>(stream_)};
  const int cap = join_first_cap(h, h->N - row0);
  const int rb = join_block_rows(h, cap, true);
  for (int64_t i0 = row0; i0 < row1; i0 += rb)
    DIRB_TRY(join_rows(R, i0, static_cast<int>(std::min<int64_t>(rb, row1 - i0)), i0, cap));
  h->join_stats[1] = h->res_off.back();
  *total_out = h->res_off.back();
  return 0;
}

int dirb200_index_join_fetch(dirb200_index* h, int64_t* off_dev, int64_t* idx_dev, double* scores_dev, void* stream_) {
  DIRB_REQUIRE(h && off_dev, DIRB200_EINVAL, "null argument");
  DIRB_REQUIRE(!h->res_off.empty(), DIRB200_ESTATE, "no range search or self-join result to fetch");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DIRB_CUDA(cudaSetDevice(h->device));
  const int64_t total = h->res_off.back();
  DIRB_CUDA(cudaMemcpyAsync(off_dev, h->res_off.data(), h->res_off.size() * 8, cudaMemcpyHostToDevice, stream));
  if (total > 0) {
    DIRB_REQUIRE(idx_dev && scores_dev, DIRB200_EINVAL, "null argument");
    DIRB_CUDA(cudaMemcpyAsync(idx_dev, h->res_ix, total * 8, cudaMemcpyDeviceToDevice, stream));
    DIRB_CUDA(cudaMemcpyAsync(scores_dev, h->res_sc, total * 8, cudaMemcpyDeviceToDevice, stream));
  }
  DIRB_CUDA(cudaStreamSynchronize(stream));    // the host offsets are the source of a copy
  return 0;
}

int dirb200_index_join_stats(dirb200_index* h, int64_t stats[5], double ms[3]) {
  DIRB_REQUIRE(h && stats && ms, DIRB200_EINVAL, "null argument");
  for (int i = 0; i < 5; ++i) stats[i] = h->join_stats[i];
  for (int i = 0; i < 3; ++i) ms[i] = h->join_ms[i];
  return 0;
}

int dirb200_index_nearest(dirb200_index* h, const float* q32_dev, int Q, int64_t* labels_dev, double* scores_dev,
                          void* stream_) {
  DIRB_REQUIRE(h && h->has_db, DIRB200_EINVAL, "index has no database");
  DIRB_TRY(no_filter(h));
  DIRB_REQUIRE(Q >= 0 && (Q == 0 || (q32_dev && labels_dev && scores_dev)), DIRB200_EINVAL, "bad arguments");
  DIRB_REQUIRE(h->N >= 1, DIRB200_EINVAL, "the index is empty");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  for (int i = 0; i < 3; ++i) h->nearest_stats[i] = 0;
  if (Q == 0) return 0;
  const int D = h->dim;
  const int64_t K = h->N;
  const int ng = static_cast<int>(ceil_div(K, 32));
  // per query: its fp16 row and its group maxima; the largest block within option ws_budget (at least 128 queries)
  const size_t per_q = static_cast<size_t>(D) * 2 + static_cast<size_t>(ng) * 4;
  const int64_t fit = static_cast<int64_t>(std::max(0.0, h->ws_budget - 4096.0) / static_cast<double>(per_q));
  const int qb = static_cast<int>(std::min<int64_t>(Q, std::max<int64_t>(128, fit / 128 * 128)));
  __half* q16;
  float* G;
  unsigned long long* st;
  auto layout = [&](void* base) {
    Carver c(base);
    q16 = c.take<__half>(static_cast<size_t>(qb) * D);
    G = c.take<float>(static_cast<size_t>(qb) * ng);
    const size_t total = c.used + 64;          // the status words, the last piece, are not rounded up
    st = c.take<unsigned long long>(8);
    return total;
  };
  DIRB_TRY(grow_ws(h, &h->ws, &h->ws_bytes, layout(nullptr)));
  layout(h->ws);
  DIRB_CUDA(cudaMemsetAsync(st, 0, 24, stream));
  for (int q0 = 0; q0 < Q; q0 += qb) {
    const int nq = std::min(qb, Q - q0);
    const float* a = q32_dev + static_cast<int64_t>(q0) * D;
    const int64_t n = static_cast<int64_t>(nq) * D;
    nearest_prep_kernel<<<static_cast<unsigned>(std::min<int64_t>(ceil_div(n, 256), 65536)), 256, 0, stream>>>(a, q16, n);
    count_launch();
    SimArgs sa;
    sa.dense = G;
    sa.dense_ld = ng;
    DIRB_TRY(sim_gemm(h, PERS_EPI_SIM_GMAX, q16, nq, h->db16, K, D, sa, stream));
    nearest_kernel<<<nq, NEAREST_THREADS, 0, stream>>>(G, ng, a, h->db32, K, D, h->eps16, h->nearest_cap, h->offset,
                                                       labels_dev + q0, scores_dev + q0, st);
    count_launch();
  }
  unsigned long long hs[3];
  DIRB_CUDA(cudaMemcpyAsync(hs, st, 24, cudaMemcpyDeviceToHost, stream));
  DIRB_CUDA(cudaStreamSynchronize(stream));
  DIRB_CUDA(cudaGetLastError());
  for (int i = 0; i < 3; ++i) h->nearest_stats[i] = static_cast<int64_t>(hs[i]);
  return 0;
}

int dirb200_index_nearest_stats(dirb200_index* h, int64_t stats[3]) {
  DIRB_REQUIRE(h && stats, DIRB200_EINVAL, "null argument");
  for (int i = 0; i < 3; ++i) stats[i] = h->nearest_stats[i];
  return 0;
}

int dirb200_topk_merge(const double* scores_dev, const int64_t* idx_dev, int G, int Q, int k, int64_t shard_stride,
                       double* out_scores_dev, int64_t* out_idx_dev, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DIRB_REQUIRE(scores_dev && idx_dev && out_scores_dev && out_idx_dev, DIRB200_EINVAL, "null argument");
  DIRB_REQUIRE(G >= 1 && Q >= 1 && k >= 1, DIRB200_EINVAL, "need G, Q, k >= 1 (got G=%d Q=%d k=%d)", G, Q, k);
  // shard g holds [Q][k] at element offset g*shard_stride, each list already ordered: rank-based merge, read in place
  if (shard_stride <= 0) shard_stride = static_cast<int64_t>(Q) * k;
  const int64_t n64 = static_cast<int64_t>(G) * k;
  if (n64 > 4096) {                          // the lists do not fit in shared memory: merge straight from global memory
    const int64_t qk = static_cast<int64_t>(Q) * k;
    fill_empty_result_kernel<<<static_cast<unsigned>(ceil_div(qk, 256)), 256, 0, stream>>>(out_scores_dev, out_idx_dev, qk);
    count_launch();
    DIRB_REQUIRE(ceil_div(n64, 256) < (int64_t(1) << 31), DIRB200_ENOTSUP, "G*k too large (G=%d k=%d)", G, k);
    merge_runs_kernel<<<dim3(static_cast<unsigned>(ceil_div(n64, 256)), std::min(Q, 65535)), 256, 0, stream>>>(
        scores_dev, idx_dev, G, k, shard_stride, k, nullptr, 0, Q, k, out_scores_dev, out_idx_dev);
    count_launch();
    DIRB_CUDA(cudaGetLastError());
    return 0;
  }
  const int n = G * k;
  const int threads = std::min(1024, (n + 31) / 32 * 32);
  merge_lists_kernel<<<Q, threads, static_cast<size_t>(n) * 16, stream>>>(scores_dev, idx_dev, G, k, shard_stride, out_scores_dev,
                                                                        out_idx_dev, PeerX{}, nullptr);
  count_launch();
  DIRB_CUDA(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------
// Peer-memory exchange of the sharded search (device side: PeerX, sel_push_kernel, search_finish_kernel, merge_lists_kernel)
struct dirb200_exchange {
  int device = 0, world = 1, rank = 0, max_q = 0, max_k = 0;
  uint8_t* base = nullptr;           // this rank's window (cudaMalloc: exportable through CUDA IPC)
  size_t bytes = 0;
  uint8_t* peer[X_MAXW] = {};        // every rank's window as mapped in this process
  bool ipc_opened[X_MAXW] = {};
  bool open = false;
  float* sel_local = nullptr;        // [max_q] this shard's selection thresholds before they are pushed
  float* seed_local = nullptr;       // [max_q] this shard's k_shard-th seed bounds before they are pushed
  unsigned long long* status = nullptr;   // status words for kernels of an empty shard (no index workspace)
};

static PeerX peer_view(const dirb200_exchange* x) {
  PeerX v{};
  v.world = x->world; v.rank = x->rank; v.max_q = x->max_q; v.max_k = x->max_k;
  for (int g = 0; g < x->world; ++g) v.peer[g] = x->peer[g];
  return v;
}

int dirb200_exchange_create(int device, int world, int rank, int max_q, int max_k, dirb200_exchange** out) {
  DIRB_REQUIRE(out, DIRB200_EINVAL, "null argument");
  DIRB_REQUIRE(world >= 1 && world <= X_MAXW && rank >= 0 && rank < world, DIRB200_ENOTSUP,
               "peer exchange supports 1..%d ranks of one box (got world=%d rank=%d)", X_MAXW, world, rank);
  DIRB_REQUIRE(max_q >= 1 && max_k >= 1 && max_k <= 1024 && static_cast<int64_t>(world) * max_k <= 4096, DIRB200_ENOTSUP,
               "need max_q >= 1, 1 <= max_k <= 1024 and world * max_k <= 4096");
  DIRB_TRY(dirb200_device_check(device));
  DIRB_CUDA(cudaSetDevice(device));
  auto* x = new dirb200_exchange();
  x->device = device; x->world = world; x->rank = rank; x->max_q = max_q; x->max_k = max_k;
  x->bytes = x_total_bytes(world, max_q, max_k);
  cudaError_t e = cudaMalloc(reinterpret_cast<void**>(&x->base), x->bytes);
  if (e == cudaSuccess) e = cudaMemset(x->base, 0, x->bytes);
  if (e == cudaSuccess) e = cudaMalloc(reinterpret_cast<void**>(&x->sel_local), static_cast<size_t>(max_q) * 4);
  if (e == cudaSuccess) e = cudaMalloc(reinterpret_cast<void**>(&x->seed_local), static_cast<size_t>(max_q) * 4);
  if (e == cudaSuccess) e = cudaMalloc(reinterpret_cast<void**>(&x->status), ST_WORDS * 8);
  if (e == cudaSuccess) e = cudaMemset(x->status, 0, ST_WORDS * 8);
  if (e == cudaSuccess) {
    const uint32_t one = 1;          // epochs start at 1: the zero-initialised flags read as "not yet published"
    e = cudaMemcpy(x->base + X_OFF_EPOCH, &one, 4, cudaMemcpyHostToDevice);
  }
  // the memsets and the pageable copy run on the legacy stream, which a search on a non-blocking stream does not wait
  // for: finish them before the window is handed out
  if (e == cudaSuccess) e = cudaStreamSynchronize(cudaStreamLegacy);
  if (e != cudaSuccess) {
    set_error("exchange window of %zu bytes: %s", x->bytes, cudaGetErrorString(e));
    dirb200_exchange_destroy(x);
    return static_cast<int>(e);
  }
  x->peer[rank] = x->base;
  *out = x;
  return 0;
}

int dirb200_exchange_ipc_handle(dirb200_exchange* x, void* handle64_out) {
  DIRB_REQUIRE(x && handle64_out, DIRB200_EINVAL, "null argument");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "CUDA IPC handles are 64 bytes");
  DIRB_CUDA(cudaSetDevice(x->device));
  cudaIpcMemHandle_t hd;
  DIRB_CUDA(cudaIpcGetMemHandle(&hd, x->base));
  memcpy(handle64_out, &hd, 64);
  return 0;
}

int dirb200_exchange_open(dirb200_exchange* x, const void* handles) {
  DIRB_REQUIRE(x && handles, DIRB200_EINVAL, "null argument");
  DIRB_REQUIRE(!x->open, DIRB200_ESTATE, "exchange already opened");
  DIRB_CUDA(cudaSetDevice(x->device));
  for (int g = 0; g < x->world; ++g) {
    if (g == x->rank) continue;
    cudaIpcMemHandle_t hd;
    memcpy(&hd, static_cast<const uint8_t*>(handles) + static_cast<size_t>(g) * 64, 64);
    void* ptr = nullptr;
    DIRB_CUDA(cudaIpcOpenMemHandle(&ptr, hd, cudaIpcMemLazyEnablePeerAccess));
    x->peer[g] = static_cast<uint8_t*>(ptr);
    x->ipc_opened[g] = true;
  }
  x->open = true;
  return 0;
}

int dirb200_exchange_open_local(dirb200_exchange* x, dirb200_exchange* const* all) {
  DIRB_REQUIRE(x && all, DIRB200_EINVAL, "null argument");
  DIRB_REQUIRE(!x->open, DIRB200_ESTATE, "exchange already opened");
  for (int g = 0; g < x->world; ++g) {
    DIRB_REQUIRE(all[g] && all[g]->world == x->world && all[g]->rank == g && all[g]->max_q == x->max_q && all[g]->max_k == x->max_k,
                 DIRB200_EINVAL, "exchange %d of the group does not match (world / rank / sizes)", g);
    if (all[g]->device != x->device) {
      int can = 0;
      DIRB_CUDA(cudaDeviceCanAccessPeer(&can, x->device, all[g]->device));
      DIRB_REQUIRE(can, DIRB200_ENOTSUP, "device %d cannot access device %d", x->device, all[g]->device);
      DIRB_CUDA(cudaSetDevice(x->device));
      cudaError_t e = cudaDeviceEnablePeerAccess(all[g]->device, 0);
      if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) DIRB_CUDA(e);
      cudaGetLastError();
    }
    x->peer[g] = all[g]->base;
  }
  x->open = true;
  return 0;
}

// Unmap the other ranks' windows (CUDA IPC).  An exporting process must not free its window while an importer still has
// it mapped: ranks call this, synchronise among themselves (a barrier), and only then destroy their own window.
int dirb200_exchange_close_peers(dirb200_exchange* x) {
  DIRB_REQUIRE(x, DIRB200_EINVAL, "null argument");
  DIRB_CUDA(cudaSetDevice(x->device));
  DIRB_CUDA(cudaDeviceSynchronize());                       // no kernel of this rank may still be writing to a peer
  for (int g = 0; g < x->world; ++g) {
    if (x->ipc_opened[g] && x->peer[g]) {
      DIRB_CUDA(cudaIpcCloseMemHandle(x->peer[g]));
      x->ipc_opened[g] = false;
    }
    if (g != x->rank) x->peer[g] = nullptr;
  }
  x->open = false;
  return 0;
}

int dirb200_exchange_destroy(dirb200_exchange* x) {
  if (!x) return 0;
  cudaSetDevice(x->device);
  for (int g = 0; g < x->world; ++g)
    if (x->ipc_opened[g] && x->peer[g]) cudaIpcCloseMemHandle(x->peer[g]);
  if (x->base) cudaFree(x->base);
  if (x->sel_local) cudaFree(x->sel_local);
  if (x->seed_local) cudaFree(x->seed_local);
  if (x->status) cudaFree(x->status);
  delete x;
  return 0;
}

int dirb200_index_search_sharded_phase(dirb200_index* h, dirb200_exchange* x, int phase, const float* q32, int Q, int k, int k_shard,
                                       double* scores_dev, int64_t* idx_dev, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DIRB_REQUIRE(h && x && q32, DIRB200_EINVAL, "null argument");
  DIRB_REQUIRE(x->open, DIRB200_ESTATE, "exchange not opened (dirb200_exchange_open / _open_local)");
  DIRB_REQUIRE(x->device == h->device, DIRB200_EINVAL, "index and exchange live on different devices");
  DIRB_REQUIRE(Q >= 1 && Q <= x->max_q && k >= 1 && k <= x->max_k, DIRB200_ENOTSUP,
               "exchange window holds %d queries x %d results (got Q=%d k=%d)", x->max_q, x->max_k, Q, k);
  const PeerX px = peer_view(x);
  const unsigned tb = static_cast<unsigned>(ceil_div(Q, 256));
  if (phase == 1) {          // queries -> fp16, seed pass; this shard's k_shard-th seed bound -> every peer's window
    DIRB_REQUIRE(k_shard >= 1 && k_shard <= k, DIRB200_EINVAL, "k_shard must be in [1, k]");
    DIRB_TRY(search_begin_seed(h, q32, Q, k, k_shard, x->sel_local, stream, x->seed_local));
    tab_push_kernel<<<tb, 256, 0, stream>>>(px, x->seed_local, Q, X_TAB_SEED, X_OFF_FSEED, 3);
    count_launch();
    DIRB_CUDA(cudaGetLastError());
    return 0;
  }
  if (phase == 2) {          // filter threshold = max(local bound, MIN of the shards' seed bounds); filter pass + selection;
                             // this shard's selection thresholds -> every peer's window
    if (h->N > 0) {
      thr_min_kernel<<<tb, 256, 0, stream>>>(px, h->pend.thr, Q, h->pend.status);
      count_launch();
    }
    DIRB_TRY(search_begin_filter(h, stream));
    tab_push_kernel<<<tb, 256, 0, stream>>>(px, x->sel_local, Q, X_TAB_SEL, X_OFF_FSEL, 0);
    count_launch();
    DIRB_CUDA(cudaGetLastError());
    return 0;
  }
  if (phase == 3)            // MIN over the shards + survivors + exact re-scoring -> ordered list into every peer's window
    return search_finish_impl(h, q32, x->sel_local, nullptr, nullptr, stream, px, x->status, false);
  DIRB_REQUIRE(phase == 4 && scores_dev && idx_dev, DIRB200_EINVAL, "phase is 1 .. 4 (4 needs the output buffers)");
  const int n = x->world * k;
  const int threads = std::min(1024, (n + 31) / 32 * 32);
  merge_lists_kernel<<<Q, threads, static_cast<size_t>(n) * 16, stream>>>(nullptr, nullptr, x->world, k, 0, scores_dev, idx_dev, px,
                                                                        h->pend.status ? h->pend.status : x->status);
  count_launch();
  DIRB_CUDA(cudaGetLastError());
  if (h->pend.status) DIRB_TRY(post_status_copy(h, stream));   // (an empty shard has no status block of its own)
  return 0;
}

int dirb200_index_search_sharded(dirb200_index* h, dirb200_exchange* x, const float* q32, int Q, int k, int k_shard,
                                 double* scores_dev, int64_t* idx_dev, void* stream_) {
  DIRB_REQUIRE(scores_dev && idx_dev, DIRB200_EINVAL, "null argument");
  for (int phase = 1; phase <= 4; ++phase)
    DIRB_TRY(dirb200_index_search_sharded_phase(h, x, phase, q32, Q, k, k_shard, scores_dev, idx_dev, stream_));
  return 0;
}

int dirb200_scores_exact(const float* q_dev, int Q, const float* db_dev, int64_t N, int D, float* out_dev,
                         void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DIRB_REQUIRE(q_dev && db_dev && out_dev && D % 4 == 0, DIRB200_EINVAL, "bad arguments");
  if (Q == 0 || N == 0) return 0;
  dim3 g(static_cast<unsigned>(ceil_div(N, 8)), static_cast<unsigned>(ceil_div(Q, 4)));
  scores_exact_kernel<<<g, 256, 0, stream>>>(q_dev, Q, db_dev, N, D, out_dev);
  count_launch();
  DIRB_CUDA(cudaGetLastError());
  return 0;
}

int dirb200_aqe_expand(const float* q_dev, int Q, int D, const float* db32_dev, const int64_t* nn_idx_dev,
                       const double* nn_scores_dev, int k, double alpha, int partial, int64_t row_offset, int64_t n_rows,
                       float* out_dev, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DIRB_REQUIRE(q_dev && nn_idx_dev && nn_scores_dev && out_dev && (db32_dev || (partial && n_rows == 0)), DIRB200_EINVAL,
               "null argument");
  DIRB_REQUIRE(k >= 1 && alpha >= 0, DIRB200_EINVAL, "k and alpha must be non-negative (test_dir.py:25)");
  if (Q == 0) return 0;
  const int kc = std::min(k, AQE_CHUNK);
  const size_t smem = static_cast<size_t>((kc + 1) & ~1) * 4 + static_cast<size_t>(kc) * 8;
  aqe_kernel<<<Q, 256, smem, stream>>>(q_dev, D, db32_dev, nn_idx_dev, nn_scores_dev, k, alpha, partial, row_offset,
                                       n_rows, out_dev);
  count_launch();
  DIRB_CUDA(cudaGetLastError());
  return 0;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------ inverted lists
// dirb200_index_search_lists (DESIGN.md section 4.10, rules I1-I6): the exact top-k of the union R(q) of the lists each
// query probes, per block of queries:
//   1. pairs (query, probed list) in (list asc, query asc) order without atomics: M[c][q] = probe rank + 1 of list c
//      for query q, one block per list counts its pairs, one block scans the lists (query segments zero-padded to a
//      multiple of 128 rows, tile offsets) and the queries (offsets of their group maxima); the totals come back to the
//      host (one synchronisation per block: the grid of the persistent passes and the workspace need them);
//   2. one block per list writes its slots (segment row -> query, first group maximum) and its tiles, m fastest
//      (CTAs running together share the list tile), and the queries are packed into their segments in fp16;
//   3. PERS_EPI_SIM_LGMAX over the tile table: the maximum of every group of 32 list rows of every pair; thr_q = k-th
//      largest of q's group maxima (distinct rows) - 2 eps16, -inf with fewer than k groups;
//   4. PERS_EPI_SIM_LFILTER over the same table into per-query candidate lists of (score, row); the counts come back to
//      the host, and a block whose lists overflowed runs again at the exact count (or in halves, rule I6);
//   5. the search's candidate selection and finish (search_finish_kernel / the deep finish) re-score against the fp32
//      rows in row order, so the key is the exact search's.
namespace dirb {
namespace {
constexpr int IVF_THREADS = 256;
constexpr int IVF_SCAN = 1024;
enum { LT_PAIRS = 0, LT_SLOTS = 1, LT_TILES = 2, LT_GROUPS = 3, LT_ROWS = 4, LT_ERR = 5, LT_MAXCNT = 6, LT_CAND = 7, LT_WORDS = 8 };

__device__ __forceinline__ int64_t list_size(const int64_t* cell_off, int c) { return cell_off[c + 1] - cell_off[c]; }

// M[c][q] = j + 1 for probe j of query q (M cleared before); a probe outside [0, K) or a list probed twice is an error.
__global__ void ivf_mark_kernel(const int64_t* __restrict__ probes, int nq, int np, int K, int* __restrict__ M,
                                long long* __restrict__ tot) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  if (i >= static_cast<int64_t>(nq) * np) return;
  const int q = static_cast<int>(i / np), j = static_cast<int>(i % np);
  const int64_t c = probes[i];
  if (c < 0 || c >= K) {
    atomicOr(reinterpret_cast<unsigned long long*>(tot + LT_ERR), 1ull);
    return;
  }
  if (atomicExch(M + c * nq + q, j + 1) != 0) atomicOr(reinterpret_cast<unsigned long long*>(tot + LT_ERR), 2ull);
}

// Per query: the offset of each probe's group maxima among the query's (probe order), their number, the probed rows.
__global__ void ivf_query_groups_kernel(const int64_t* __restrict__ probes, int nq, int np, int K,
                                        const int64_t* __restrict__ cell_off, int* __restrict__ loc,
                                        long long* __restrict__ qgroups, long long* __restrict__ tot) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= nq) return;
  long long g = 0, rows = 0;
  for (int j = 0; j < np; ++j) {
    const int64_t c = probes[static_cast<int64_t>(q) * np + j];
    loc[static_cast<int64_t>(q) * np + j] = static_cast<int>(g);
    if (c < 0 || c >= K) continue;
    const int64_t n = list_size(cell_off, static_cast<int>(c));
    g += (n + 31) / 32;
    rows += n;
  }
  qgroups[q] = g;
  atomicAdd(reinterpret_cast<unsigned long long*>(tot + LT_ROWS), static_cast<unsigned long long>(rows));
}

// One block per list: its number of probing queries.
__global__ void __launch_bounds__(IVF_THREADS) ivf_list_count_kernel(const int* __restrict__ M, int nq, int* __restrict__ pc) {
  __shared__ int red[IVF_THREADS / 32];
  const int c = blockIdx.x;
  int n = 0;
  for (int q = threadIdx.x; q < nq; q += IVF_THREADS) n += M[static_cast<int64_t>(c) * nq + q] != 0;
  for (int o = 16; o > 0; o >>= 1) n += __shfl_xor_sync(0xffffffffu, n, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = n;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < IVF_THREADS / 32; ++w) n += red[w];
    pc[c] = n;
  }
}

// One block: segment and tile offsets of the lists (lists without rows get neither), group offsets of the queries.
__global__ void __launch_bounds__(IVF_SCAN) ivf_scan_kernel(const int* __restrict__ pc, const int64_t* __restrict__ cell_off, int K,
                                                           const long long* __restrict__ qgroups, int nq,
                                                           int64_t* __restrict__ seg_off, int64_t* __restrict__ tile_off,
                                                           int64_t* __restrict__ qgoff, long long* __restrict__ tot) {
  __shared__ long long ws[IVF_SCAN / 32];
  long long cs = 0, ct = 0, cp = 0;
  for (int base = 0; base < K; base += IVF_SCAN) {
    const int c = base + threadIdx.x;
    long long slots = 0, tiles = 0, pairs = 0;
    if (c < K) {
      const int64_t n = list_size(cell_off, c);
      pairs = pc[c];
      if (n > 0) {
        slots = (pairs + 127) / 128 * 128;
        tiles = slots / 128 * ((n + 127) / 128);
      }
    }
    long long t1, t2, t3;
    const long long is = block_scan(slots, ws, &t1);
    const long long it = block_scan(tiles, ws, &t2);
    block_scan(pairs, ws, &t3);
    if (c < K) {
      seg_off[c] = cs + is - slots;
      tile_off[c] = ct + it - tiles;
    }
    cs += t1;
    ct += t2;
    cp += t3;
  }
  long long cg = 0;
  for (int base = 0; base < nq; base += IVF_SCAN) {
    const int q = base + threadIdx.x;
    const long long v = q < nq ? qgroups[q] : 0;
    long long t;
    const long long incl = block_scan(v, ws, &t);
    if (q < nq) qgoff[q] = cg + incl - v;
    cg += t;
  }
  if (threadIdx.x == 0) {
    seg_off[K] = cs;
    tile_off[K] = ct;
    qgoff[nq] = cg;
    tot[LT_PAIRS] = cp;
    tot[LT_SLOTS] = cs;
    tot[LT_TILES] = ct;
    tot[LT_GROUPS] = cg;
  }
}

// One block per list with rows: its slots in ascending query order (a block-wide scan of M[c][*]), the zero padding of
// its segment, and its tiles {A row, B row, column tile, valid rows | valid columns << 16}, m fastest.
__global__ void __launch_bounds__(IVF_THREADS) ivf_list_fill_kernel(const int* __restrict__ M, int nq, int np,
                                                                   const int* __restrict__ pc,
                                                                   const int64_t* __restrict__ cell_off,
                                                                   const int64_t* __restrict__ seg_off,
                                                                   const int64_t* __restrict__ tile_off,
                                                                   const int64_t* __restrict__ qgoff, const int* __restrict__ loc,
                                                                   int* __restrict__ slot_q, int64_t* __restrict__ gbase,
                                                                   int4* __restrict__ tiles) {
  __shared__ long long ws[IVF_THREADS / 32];
  const int c = blockIdx.x;
  const int64_t n = list_size(cell_off, c);
  const int pairs = pc[c];
  if (n == 0 || pairs == 0) return;
  const int64_t s0 = seg_off[c];
  long long carry = 0;
  for (int base = 0; base < nq; base += IVF_THREADS) {
    const int q = base + threadIdx.x;
    const int j1 = q < nq ? M[static_cast<int64_t>(c) * nq + q] : 0;
    long long t;
    const long long incl = block_scan<long long>(j1 != 0, ws, &t);
    if (j1 != 0) {
      const int64_t s = s0 + carry + incl - 1;
      slot_q[s] = q;
      gbase[s] = qgoff[q] + loc[static_cast<int64_t>(q) * np + j1 - 1];
    }
    carry += t;
  }
  const int slots = (pairs + 127) / 128 * 128;
  for (int s = pairs + threadIdx.x; s < slots; s += IVF_THREADS) {
    slot_q[s0 + s] = -1;
    gbase[s0 + s] = 0;
  }
  const int mt = slots / 128;
  const int nt = static_cast<int>((n + 127) / 128);
  const int64_t t0 = tile_off[c];
  for (int i = threadIdx.x; i < mt * nt; i += IVF_THREADS) {
    const int m = i % mt, nn = i / mt;
    const int mv = min(128, pairs - 128 * m);
    const int64_t left = n - 128 * static_cast<int64_t>(nn);
    const int nv = left < 128 ? static_cast<int>(left) : 128;
    tiles[t0 + i] = make_int4(static_cast<int>(s0 + 128 * m), static_cast<int>(cell_off[c] + 128 * static_cast<int64_t>(nn)), nn,
                              mv | (nv << 16));
  }
}

// Packed fp16 queries: slot s holds query slot_q[s], padding slots zeros.  Candidate counters cleared.
__global__ void ivf_pack_kernel(const float* __restrict__ q32, int D, const int* __restrict__ slot_q, int64_t slots,
                                __half* __restrict__ q16, int* __restrict__ cnt, int nq) {
  const int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x;
  const int d4 = D / 4;
  if (i < nq) cnt[i] = 0;
  if (i >= slots * d4) return;
  const int64_t s = i / d4;
  const int d = static_cast<int>(i % d4) * 4;
  const int q = slot_q[s];
  uint2 o = make_uint2(0u, 0u);
  if (q >= 0) {
    const float4 v = *reinterpret_cast<const float4*>(q32 + static_cast<int64_t>(q) * D + d);
    o.x = pack_h2(v.x, v.y);
    o.y = pack_h2(v.z, v.w);
  }
  *reinterpret_cast<uint2*>(q16 + s * D + d) = o;
}

// thr[q] = (k-th largest of the query's group maxima) - band; fewer than k groups -> -inf.
__global__ void __launch_bounds__(SEL_THREADS) ivf_seed_kernel(const float* __restrict__ G, const int64_t* __restrict__ qgoff,
                                                               int k, float band, float* __restrict__ thr) {
  __shared__ uint32_t hist[256];
  __shared__ uint32_t bc[2];
  const int q = blockIdx.x;
  const int64_t g0 = qgoff[q];
  const float t = block_kth_largest(DenseAcc{G + g0}, static_cast<int>(qgoff[q + 1] - g0), k, hist, bc);
  if (threadIdx.x == 0) thr[q] = t - band;
}

// Largest candidate count (the exact size a re-run needs) and the candidates captured in all.
__global__ void ivf_count_kernel(const int* __restrict__ cnt, int nq, long long* __restrict__ tot) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= nq) return;
  atomicMax(tot + LT_MAXCNT, static_cast<long long>(cnt[q]));
  atomicAdd(reinterpret_cast<unsigned long long*>(tot + LT_CAND), static_cast<unsigned long long>(cnt[q]));
}
}  // namespace
}  // namespace dirb

// List search of nq queries probing np of K lists, part 1 (lws[0]): the (list, query) pair marks and per-query list
// positions, the pair counts and offsets, and the table totals.  It survives the re-runs of part 2.
struct ListPairWs {
  int *M, *loc, *pc;
  long long *qgroups, *tot;
  int64_t *seg_off, *tile_off, *qgoff;
  size_t total;
};
static ListPairWs list_pair_ws(void* base, int K, int nq, int np) {
  Carver c(base);
  ListPairWs w;
  w.M = c.take<int>(static_cast<size_t>(K) * nq);
  w.loc = c.take<int>(static_cast<size_t>(nq) * np);
  w.qgroups = c.take<long long>(nq);
  w.pc = c.take<int>(K);
  w.seg_off = c.take<int64_t>(static_cast<size_t>(K) + 1);
  w.tile_off = c.take<int64_t>(static_cast<size_t>(K) + 1);
  w.qgoff = c.take<int64_t>(static_cast<size_t>(nq) + 1);
  w.tot = c.take<long long>(LT_WORDS);
  w.total = c.used;
  return w;
}

// Part 2 (lws[1]): the tile table, packed queries, group maxima, candidate lists and the finish's buffers.
struct ListWs {
  __half* q16;
  int *slot_q, *cnt, *gates, *surv_cnt = nullptr;
  int64_t* gbase;
  int4* tiles;
  float *G, *thr, *kth_k, *sel;
  unsigned long long *cand, *status;
  SortScratch surv{};
  size_t total;
};
static ListWs list_ws(void* base, int64_t slots, int64_t n_tiles, int64_t groups, int D, int nq, int cap,
                      const SearchSizes& z) {
  Carver c(base);
  ListWs w;
  w.q16 = c.take<__half>(static_cast<size_t>(slots) * D);
  w.slot_q = c.take<int>(slots);
  w.gbase = c.take<int64_t>(slots);
  w.tiles = c.take<int4>(n_tiles);
  w.G = c.take<float>(groups);
  w.thr = c.take<float>(nq);
  w.cnt = c.take<int>(nq);
  w.cand = c.take<unsigned long long>(static_cast<size_t>(nq) * cap);
  w.kth_k = c.take<float>(nq);
  w.sel = c.take<float>(nq);
  w.gates = c.take<int>(8);
  w.status = c.take<unsigned long long>(ST_WORDS);
  if (z.deep) {
    w.surv = take_sort_scratch(c, nq, z.cap2);
    w.surv_cnt = c.take<int>(nq);
  }
  w.total = c.used;
  return w;
}

// One block of nq queries.  *split = 1: the block's workspace does not fit option ws_budget (nothing was written).
static int lists_block(dirb200_index* h, const float* q32, int nq, int k, const int64_t* probes, int np, double* out_sc,
                       int64_t* out_ix, cudaStream_t stream, int* split) {
  const int K = h->lists_k, D = h->dim;
  const int64_t N = h->N;
  *split = 0;
  // ---- 1. pair counts and offsets
  const size_t bytesA = list_pair_ws(nullptr, K, nq, np).total;
  if (nq > 1 && static_cast<double>(bytesA) > h->ws_budget) { *split = 1; return 0; }
  DIRB_TRY(grow_ws(h, &h->lws[0], &h->lws_bytes[0], bytesA));
  const ListPairWs pw = list_pair_ws(h->lws[0], K, nq, np);
  if (h->profile) h->lev.mark(0, stream);
  DIRB_CUDA(cudaMemsetAsync(pw.M, 0, static_cast<size_t>(K) * nq * 4, stream));
  DIRB_CUDA(cudaMemsetAsync(pw.tot, 0, LT_WORDS * 8, stream));
  const int64_t npairs = static_cast<int64_t>(nq) * np;
  ivf_mark_kernel<<<static_cast<unsigned>(ceil_div(npairs, IVF_THREADS)), IVF_THREADS, 0, stream>>>(probes, nq, np, K, pw.M, pw.tot);
  ivf_query_groups_kernel<<<static_cast<unsigned>(ceil_div(nq, IVF_THREADS)), IVF_THREADS, 0, stream>>>(
      probes, nq, np, K, h->lcell_off, pw.loc, pw.qgroups, pw.tot);
  ivf_list_count_kernel<<<K, IVF_THREADS, 0, stream>>>(pw.M, nq, pw.pc);
  ivf_scan_kernel<<<1, IVF_SCAN, 0, stream>>>(pw.pc, h->lcell_off, K, pw.qgroups, nq, pw.seg_off, pw.tile_off, pw.qgoff, pw.tot);
  count_launch(4);
  long long ht[LT_WORDS];
  DIRB_CUDA(cudaMemcpyAsync(ht, pw.tot, sizeof(ht), cudaMemcpyDeviceToHost, stream));
  DIRB_CUDA(cudaStreamSynchronize(stream));
  DIRB_CUDA(cudaGetLastError());
  DIRB_REQUIRE((ht[LT_ERR] & 1) == 0, DIRB200_EINVAL, "a probe lies outside [0, %d)", K);
  DIRB_REQUIRE((ht[LT_ERR] & 2) == 0, DIRB200_EINVAL, "a query probes the same list twice");
  const int64_t slots = ht[LT_SLOTS], n_tiles = ht[LT_TILES], groups = ht[LT_GROUPS];
  // ---- 2.-5. per candidate capacity: first the default, then (rule I6) the exact largest count
  const SearchSizes z = search_sizes(h, k);
  int cap = h->cand_cap > 0 ? h->cand_cap : z.cap;
  const int cap2 = z.cap2;
  const float band = static_cast<float>(2.0 * h->eps16);
  for (int run = 0;; ++run) {
    const size_t bytesB = list_ws(nullptr, slots, n_tiles, groups, D, nq, cap, z).total;
    if (static_cast<double>(bytesA + bytesB) > h->ws_budget) {
      if (nq > 1) { *split = 1; return 0; }
      DIRB_REQUIRE(false, DIRB200_EOVERFLOW,
                   "the list search of one query needs %.0f bytes (%d candidates) and option ws_budget is %.0f bytes",
                   static_cast<double>(bytesA + bytesB), cap, h->ws_budget);
    }
    DIRB_TRY(grow_ws(h, &h->lws[1], &h->lws_bytes[1], bytesB));
    const ListWs w = list_ws(h->lws[1], slots, n_tiles, groups, D, nq, cap, z);
    if (run > 0 && h->profile) h->lev.mark(0, stream);
    ivf_list_fill_kernel<<<K, IVF_THREADS, 0, stream>>>(pw.M, nq, np, pw.pc, h->lcell_off, pw.seg_off, pw.tile_off, pw.qgoff,
                                                         pw.loc, w.slot_q, w.gbase, w.tiles);
    const int64_t packs = std::max<int64_t>(slots * (D / 4), nq);
    ivf_pack_kernel<<<static_cast<unsigned>(ceil_div(packs, IVF_THREADS)), IVF_THREADS, 0, stream>>>(q32, D, w.slot_q, slots,
                                                                                                     w.q16, w.cnt, nq);
    DIRB_CUDA(cudaMemsetAsync(w.gates, 0, 8 * 4, stream));
    DIRB_CUDA(cudaMemsetAsync(w.status, 0, ST_WORDS * 8, stream));
    DIRB_CUDA(cudaMemsetAsync(pw.tot + LT_MAXCNT, 0, 16, stream));
    count_launch(2);
    if (h->profile) h->lev.mark(1, stream);
    SimArgs a;
    a.tiles = w.tiles;
    a.n_tiles = n_tiles;
    a.slot_q = w.slot_q;
    a.gbase = w.gbase;
    if (n_tiles > 0) {
      a.dense = w.G;
      DIRB_TRY(sim_gemm(h, PERS_EPI_SIM_LGMAX, w.q16, slots, h->l16, N, D, a, stream));
    }
    ivf_seed_kernel<<<nq, SEL_THREADS, 0, stream>>>(w.G, pw.qgoff, k, band, w.thr);
    count_launch();
    if (h->profile) h->lev.mark(2, stream);
    if (n_tiles > 0) {
      a.dense = nullptr;
      a.thr = w.thr;
      a.cand = w.cand;
      a.cand_cnt = w.cnt;
      a.cand_cap = cap;
      DIRB_TRY(sim_gemm(h, PERS_EPI_SIM_LFILTER, w.q16, slots, h->l16, N, D, a, stream));
    }
    ivf_count_kernel<<<static_cast<unsigned>(ceil_div(nq, IVF_THREADS)), IVF_THREADS, 0, stream>>>(w.cnt, nq, pw.tot);
    count_launch();
    DIRB_CUDA(cudaMemcpyAsync(ht + LT_MAXCNT, pw.tot + LT_MAXCNT, 16, cudaMemcpyDeviceToHost, stream));
    DIRB_CUDA(cudaStreamSynchronize(stream));
    DIRB_CUDA(cudaGetLastError());
    if (ht[LT_MAXCNT] > cap) {               // rule I6: run the block again with room for every match
      DIRB_REQUIRE(ht[LT_MAXCNT] < (int64_t(1) << 30), DIRB200_EOVERFLOW, "%lld candidates for one query",
                   static_cast<long long>(ht[LT_MAXCNT]));
      cap = static_cast<int>((ht[LT_MAXCNT] + 255) / 256 * 256);
      ++h->lists_stats[5];
      continue;
    }
    cand_kth_kernel<<<nq, SEL_THREADS, 0, stream>>>(w.cand, w.cnt, cap, k, k, band, w.kth_k, w.sel, w.thr, N, nullptr, w.gates,
                                                    1, w.status);
    count_launch();
    if (h->profile) h->lev.mark(3, stream);
    auto& P = h->pend;
    P = dirb200_index::Pending();
    P.active = true;
    P.Q = nq;
    P.k = k;
    P.cap = cap;
    P.cap2 = cap2;
    P.band = band;
    P.cnt = w.cnt;
    P.cand = w.cand;
    P.status = w.status;
    P.kth_k = w.kth_k;
    P.sel_dev = w.sel;
    P.launches0 = launches_total();
    P.surv = w.surv;
    P.surv_cnt = w.surv_cnt;
    DIRB_TRY(search_finish_impl(h, q32, w.sel, out_sc, out_ix, stream, PeerX{}, nullptr, true));
    if (h->profile) h->lev.mark(4, stream);
    h->lists_stats[0] += ht[LT_PAIRS];
    h->lists_stats[1] += slots;
    h->lists_stats[2] += n_tiles;
    h->lists_stats[3] += ht[LT_ROWS];
    h->lists_stats[4] += ht[LT_CAND];
    if (h->profile) {
      DIRB_CUDA(cudaEventSynchronize(h->lev.ev[4]));
      for (int i = 0; i < 4; ++i) h->lists_ms[i] += h->lev.ms(i, i + 1);
    }
    return 0;
  }
}

extern "C" {

int dirb200_index_set_lists(dirb200_index* h, const void* db16_lists_dev, const int64_t* perm_dev, const int64_t* cell_off_dev,
                            int K, void* stream_) {
  DIRB_REQUIRE(h && h->has_db, DIRB200_ESTATE, "index has no database attached");
  DIRB_REQUIRE(K >= 0, DIRB200_EINVAL, "K must be >= 0");
  h->tmaps.es.clear();
  h->l16 = nullptr;
  h->lperm = nullptr;
  h->lcell_off = nullptr;
  h->lists_k = 0;
  if (K == 0) return 0;                       // detaches the lists
  DIRB_REQUIRE(h->N >= 1 && db16_lists_dev && perm_dev && cell_off_dev, DIRB200_EINVAL, "bad list arguments");
  DIRB_CUDA(cudaSetDevice(h->device));
  std::vector<int64_t> off(static_cast<size_t>(K) + 1);
  DIRB_CUDA(cudaMemcpyAsync(off.data(), cell_off_dev, off.size() * 8, cudaMemcpyDeviceToHost, static_cast<cudaStream_t>(stream_)));
  DIRB_CUDA(cudaStreamSynchronize(static_cast<cudaStream_t>(stream_)));
  DIRB_REQUIRE(off[0] == 0 && off[K] == h->N, DIRB200_EINVAL, "cell offsets must run from 0 to N = %lld",
               static_cast<long long>(h->N));
  for (int c = 0; c < K; ++c) DIRB_REQUIRE(off[c] <= off[c + 1], DIRB200_EINVAL, "cell offsets must not decrease (list %d)", c);
  h->l16 = static_cast<const __half*>(db16_lists_dev);
  h->lperm = perm_dev;
  h->lcell_off = cell_off_dev;
  h->lists_k = K;
  return 0;
}

int dirb200_index_search_lists(dirb200_index* h, const float* q32_dev, int Q, int k, const int64_t* probes_dev, int nprobe,
                               double* scores_dev, int64_t* idx_dev, void* stream_) {
  DIRB_REQUIRE(h && h->lists_k > 0, DIRB200_ESTATE, "index has no lists attached (dirb200_index_set_lists)");
  DIRB_TRY(no_filter(h));
  DIRB_REQUIRE(Q >= 0 && (Q == 0 || (q32_dev && probes_dev && scores_dev && idx_dev)), DIRB200_EINVAL, "bad arguments");
  DIRB_REQUIRE(k >= 1 && k <= K_MAX, DIRB200_ENOTSUP, "need 0 < k <= %d (got %d)", K_MAX, k);
  DIRB_REQUIRE(nprobe >= 1 && nprobe <= h->lists_k, DIRB200_EINVAL, "nprobe must be in [1, %d] (got %d)", h->lists_k, nprobe);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  for (auto& v : h->lists_stats) v = 0;
  for (auto& v : h->lists_ms) v = 0;
  if (Q == 0) return 0;
  DIRB_CUDA(cudaSetDevice(h->device));
  DIRB_TRY(dirb200_index_check(h));
  // blocks start at the exact search's size and are halved while their workspace does not fit (rule I6)
  int qb = std::min(Q, search_max_queries(h, k));
  for (int q0 = 0; q0 < Q;) {
    const int nb = std::min(qb, Q - q0);
    int split = 0;
    DIRB_TRY(lists_block(h, q32_dev + static_cast<int64_t>(q0) * h->dim, nb, k, probes_dev + static_cast<int64_t>(q0) * nprobe,
                         nprobe, scores_dev + static_cast<int64_t>(q0) * k, idx_dev + static_cast<int64_t>(q0) * k, stream, &split));
    if (split) {
      qb = (nb + 1) / 2;
      continue;
    }
    q0 += nb;
  }
  return 0;
}

int dirb200_index_lists_stats(dirb200_index* h, int64_t stats[6], double ms[4]) {
  DIRB_REQUIRE(h && stats && ms, DIRB200_EINVAL, "null argument");
  for (int i = 0; i < 6; ++i) stats[i] = h->lists_stats[i];
  for (int i = 0; i < 4; ++i) ms[i] = h->lists_ms[i];
  return 0;
}

}  // extern "C"
