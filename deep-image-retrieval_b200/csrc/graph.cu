// Graph search over a pruned kNN graph of the database (DESIGN.md section 4.12, rules G1-G8).
//
//   graph_prune_kernel   G3 / G4: one CTA per row r.  knn(r) and its neighbours' lists sit in shared memory; thread j
//                        counts the detours of position j, then block_bitonic_sort orders (detours, position) keys and
//                        the first `degree` give F(r).
//   graph_merge_kernel   G5: one warp per row.  F(r)[0 : degree/2], then Rev(r) (ordered outside, by a stable sort of
//                        (target, position) keys over the entries in source order), then the rest of F(r), each entry
//                        appended unless the warp finds it already present.
//   graph_search_kernel  G7: one CTA per query.  The visited set V is an open-addressing table of rows in shared memory
//                        with at least twice as many slots as V can hold, so an insertion always finds a slot and V is
//                        a set whatever order the atomicCASes take.  Each iteration picks the parents with a block scan
//                        over B's expanded flags, looks the parents' graph entries up in V, finds the first
//                        (parent, edge) slot of each new row through a second table (atomicMin on (row, slot) keys),
//                        keeps that slot and compacts the kept ones in slot order with a block scan (so N_t's order
//                        does not depend on scheduling), scores the new rows with exact_dot_warp (one warp per row),
//                        sorts them with block_bitonic_sort and merges them into B by rank_in_run.
#include <math.h>
#include <stdint.h>

#include <algorithm>

#include "block.cuh"
#include "common.h"
#include "exact_dot.cuh"

namespace dirb {
namespace {

constexpr int GRAPH_MAX_K = 128;         // longest kNN list (build_k)
constexpr int GRAPH_MAX_DEGREE = 128;
constexpr int PRUNE_THREADS = 128;
constexpr int MERGE_WARPS = 8;
constexpr int GS_THREADS = 512;
constexpr int GS_WARPS = GS_THREADS / 32;

size_t prune_smem(int K) { return static_cast<size_t>(K) * (K + 1) * sizeof(int); }

__host__ __device__ inline int pow2_at_least(int64_t n) {
  int p = 1;
  while (p < n) p <<= 1;
  return p;
}

// The search's dynamic shared memory: B twice (scores, rows, expanded flags), the batch of new rows (P entries, a
// power of two, for the sort), the table of first (parent, edge) slots (2^log2F >= 2W entries), the visited table
// (S slots), the (parent, edge) slots and the parents.  Offsets in bytes; every array starts 8-byte aligned.
struct GsLayout {
  int log2S, log2F, P, W;
  size_t bsc[2], bix[2], bex[2], nsc, nix, first, hash, cand, par, total;
};
__host__ __device__ inline GsLayout gs_layout(int n_seeds, int itopk, int width, int degree, int max_iter) {
  GsLayout l;
  const int64_t cap = static_cast<int64_t>(n_seeds) + static_cast<int64_t>(max_iter) * width * degree;
  l.log2S = 1;
  while ((int64_t(1) << l.log2S) < 2 * cap) ++l.log2S;
  l.W = width * degree;
  l.log2F = 1;
  while ((1 << l.log2F) < 2 * l.W) ++l.log2F;
  l.P = pow2_at_least(std::max(n_seeds, l.W));
  size_t o = 0;
  auto take = [&](size_t bytes) {
    const size_t at = o;
    o += (bytes + 7) / 8 * 8;
    return at;
  };
  for (int b = 0; b < 2; ++b) {
    l.bsc[b] = take(static_cast<size_t>(itopk) * sizeof(double));
    l.bix[b] = take(static_cast<size_t>(itopk) * sizeof(int64_t));
  }
  l.nsc = take(static_cast<size_t>(l.P) * sizeof(double));
  l.nix = take(static_cast<size_t>(l.P) * sizeof(int64_t));
  l.first = take((size_t(1) << l.log2F) * sizeof(unsigned long long));
  for (int b = 0; b < 2; ++b) l.bex[b] = take(static_cast<size_t>(itopk) * sizeof(int));
  l.hash = take((size_t(1) << l.log2S) * sizeof(int));
  l.cand = take(static_cast<size_t>(l.W) * sizeof(int));
  l.par = take(static_cast<size_t>(width) * sizeof(int));
  l.total = o;
  return l;
}

// knn [n][K] int32 (r removed, -1 entries allowed) -> F [n][degree] int32, -1 padded.
__global__ void __launch_bounds__(PRUNE_THREADS) graph_prune_kernel(const int* __restrict__ knn, int K, int degree,
                                                                    int* __restrict__ fwd) {
  extern __shared__ int psm[];
  __shared__ uint32_t key[GRAPH_MAX_K];
  int* L = psm;           // [K]   knn(r)
  int* NL = psm + K;      // [K][K] knn(n_i), -1 rows for n_i = -1
  const int64_t r = blockIdx.x;
  for (int j = threadIdx.x; j < K; j += PRUNE_THREADS) L[j] = knn[r * K + j];
  __syncthreads();
  for (int e = threadIdx.x; e < K * K; e += PRUNE_THREADS) {
    const int i = e / K, p = e - i * K, ni = L[i];
    NL[e] = ni >= 0 ? knn[static_cast<int64_t>(ni) * K + p] : -1;
  }
  __syncthreads();
  const int P = pow2_at_least(K);
  for (int j = threadIdx.x; j < P; j += PRUNE_THREADS) {
    uint32_t kj = 0xffffffffu;
    const int nj = j < K ? L[j] : -1;
    if (nj >= 0) {
      // G3: the i < j whose own list holds n_j before position j
      uint32_t det = 0;
      for (int i = 0; i < j; ++i) {
        const int* li = NL + i * K;
        bool hit = false;
        for (int p = 0; p < j; ++p) hit |= li[p] == nj;
        det += hit;
      }
      kj = (det << 8) | static_cast<uint32_t>(j);
    }
    key[j] = kj;
  }
  __syncthreads();
  block_bitonic_sort<PRUNE_THREADS>(key, P, [](uint32_t a, uint32_t b) { return a < b; });
  for (int t = threadIdx.x; t < degree; t += PRUNE_THREADS)
    fwd[r * degree + t] = t < P && key[t] != 0xffffffffu ? L[key[t] & 255u] : -1;
}

// F [n][degree], Rev as a CSR (rev_off [n + 1], rev_src in (position, source) order per target) -> G [n][degree].
__global__ void __launch_bounds__(MERGE_WARPS * 32) graph_merge_kernel(const int* __restrict__ fwd, int64_t n, int degree,
                                                                       const int64_t* __restrict__ rev_off,
                                                                       const int* __restrict__ rev_src,
                                                                       int* __restrict__ graph) {
  __shared__ int gs[MERGE_WARPS][GRAPH_MAX_DEGREE];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t r = static_cast<int64_t>(blockIdx.x) * MERGE_WARPS + w;
  if (r >= n) return;
  int* g = gs[w];
  const int* f = fwd + r * degree;
  int nf = 0;
  for (int t = lane; t < degree; t += 32) nf += f[t] >= 0;
  nf = __reduce_add_sync(0xffffffffu, nf);
  int cnt = min(degree / 2, nf);
  for (int t = lane; t < cnt; t += 32) g[t] = f[t];
  __syncwarp();
  auto add = [&](int c) {
    bool dup = false;
    for (int t = lane; t < cnt; t += 32) dup |= g[t] == c;
    if (!__any_sync(0xffffffffu, dup)) {
      if (lane == 0) g[cnt] = c;
      ++cnt;
    }
    __syncwarp();
  };
  // at most degree / 2 reverse entries are already present (Rev(r) holds each source once), so this loop ends
  for (int64_t e = rev_off[r]; e < rev_off[r + 1] && cnt < degree; ++e) add(rev_src[e]);
  for (int t = degree / 2; t < nf && cnt < degree; ++t) add(f[t]);
  for (int t = lane; t < degree; t += 32) graph[r * degree + t] = t < cnt ? g[t] : -1;
}

__device__ __forceinline__ uint32_t gs_hash(int c, int log2S) {
  return (static_cast<uint32_t>(c) * 2654435761u) >> (32 - log2S);
}
__device__ __forceinline__ bool gs_lookup(const int* H, uint32_t mask, int log2S, int c) {
  for (uint32_t h = gs_hash(c, log2S);; h = (h + 1) & mask) {
    const int v = H[h];
    if (v == c) return true;
    if (v < 0) return false;
  }
}
__device__ __forceinline__ void gs_insert(int* H, uint32_t mask, int log2S, int c) {
  for (uint32_t h = gs_hash(c, log2S);; h = (h + 1) & mask) {
    const int old = atomicCAS(H + h, -1, c);
    if (old < 0 || old == c) return;
  }
}

template <class T>
__device__ __forceinline__ void swap_ptr(T*& a, T*& b) {
  T* t = a;
  a = b;
  b = t;
}

// The first-slot table: one entry (row << 32 | slot) per row of the iteration's (parent, edge) slots, holding the
// smallest slot that names the row whatever order the atomics take.
constexpr unsigned long long GS_FREE = ~0ull;
__device__ __forceinline__ void first_slot_note(unsigned long long* F, uint32_t mask, int log2F, int c, int slot) {
  const unsigned long long key = (static_cast<unsigned long long>(c) << 32) | static_cast<uint32_t>(slot);
  for (uint32_t h = gs_hash(c, log2F);; h = (h + 1) & mask) {
    const unsigned long long old = atomicCAS(F + h, GS_FREE, key);
    if (old == GS_FREE) return;
    if ((old >> 32) == static_cast<unsigned long long>(c)) {
      atomicMin(F + h, key);
      return;
    }
  }
}
__device__ __forceinline__ int first_slot(const unsigned long long* F, uint32_t mask, int log2F, int c) {
  for (uint32_t h = gs_hash(c, log2F);; h = (h + 1) & mask)
    if ((F[h] >> 32) == static_cast<unsigned long long>(c)) return static_cast<int>(F[h] & 0xffffffffu);
}

__global__ void __launch_bounds__(GS_THREADS, 1) graph_search_kernel(
    const float* __restrict__ q, int D, const float* __restrict__ x, const int* __restrict__ graph, int degree,
    const int* __restrict__ seeds, int n_seeds, int itopk, int width, int max_iter, int k,
    double* __restrict__ out_s, int64_t* __restrict__ out_i, int64_t* __restrict__ vis_rows,
    double* __restrict__ vis_sc, int64_t vcap, int* __restrict__ n_vis, int* __restrict__ n_iter) {
  extern __shared__ __align__(16) unsigned char gsm[];
  __shared__ int warp_sums[GS_WARPS];
  const GsLayout l = gs_layout(n_seeds, itopk, width, degree, max_iter);
  // B is double-buffered: (bs, bi, be) the current buffer, (ts, ti, te) the one the next merge writes
  double* bs = reinterpret_cast<double*>(gsm + l.bsc[0]);
  int64_t* bi = reinterpret_cast<int64_t*>(gsm + l.bix[0]);
  int* be = reinterpret_cast<int*>(gsm + l.bex[0]);
  double* ts = reinterpret_cast<double*>(gsm + l.bsc[1]);
  int64_t* ti = reinterpret_cast<int64_t*>(gsm + l.bix[1]);
  int* te = reinterpret_cast<int*>(gsm + l.bex[1]);
  double* nsc = reinterpret_cast<double*>(gsm + l.nsc);
  int64_t* nix = reinterpret_cast<int64_t*>(gsm + l.nix);
  int* H = reinterpret_cast<int*>(gsm + l.hash);
  int* cand = reinterpret_cast<int*>(gsm + l.cand);
  unsigned long long* F = reinterpret_cast<unsigned long long*>(gsm + l.first);
  const uint32_t fmask = (1u << l.log2F) - 1u;
  int* par = reinterpret_cast<int*>(gsm + l.par);
  const uint32_t mask = (1u << l.log2S) - 1u;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t qi = blockIdx.x;
  const float* qrow = q + qi * D;

  for (uint32_t h = threadIdx.x; h <= mask; h += GS_THREADS) H[h] = -1;
  for (uint32_t h = threadIdx.x; h <= fmask; h += GS_THREADS) F[h] = GS_FREE;
  for (int i = threadIdx.x; i < itopk; i += GS_THREADS) {
    bs[i] = ts[i] = -INFINITY;
    bi[i] = ti[i] = -1;
    be[i] = te[i] = 1;
  }
  __syncthreads();
  // the seeds are the first batch: distinct rows (G6), inserted as they are
  for (int j = threadIdx.x; j < n_seeds; j += GS_THREADS) {
    const int c = seeds[qi * n_seeds + j];
    nix[j] = c;
    gs_insert(H, mask, l.log2S, c);
  }
  int nn = n_seeds, nB = 0, it = 0;
  int64_t nv = 0;
  __syncthreads();
  for (;;) {
    // score the batch (arrival order), record it, sort it and merge it into B
    for (int j = warp; j < nn; j += GS_WARPS) {
      const double e = exact_dot_warp(qrow, x + nix[j] * D, D, lane);
      if (lane == 0) nsc[j] = e;
    }
    const int P = pow2_at_least(nn);
    for (int j = nn + threadIdx.x; j < P; j += GS_THREADS) {
      nsc[j] = -INFINITY;
      nix[j] = INT64_MAX;
    }
    __syncthreads();
    if (vis_rows) {
      for (int j = threadIdx.x; j < nn; j += GS_THREADS) {
        vis_rows[qi * vcap + nv + j] = nix[j];
        vis_sc[qi * vcap + nv + j] = nsc[j];
      }
      __syncthreads();
    }
    block_bitonic_sort<GS_THREADS>(nsc, nix, P, [](double sa, int64_t ia, double sb, int64_t ib) {
      return ranks_before(sa, ia, sb, ib);
    });
    const auto ld = [](auto p) { return *p; };
    for (int i = threadIdx.x; i < nB; i += GS_THREADS) {
      const int pos = i + rank_in_run(nsc, nix, nn, bs[i], bi[i], ld);
      if (pos < itopk) {
        ts[pos] = bs[i];
        ti[pos] = bi[i];
        te[pos] = be[i];
      }
    }
    for (int j = threadIdx.x; j < nn; j += GS_THREADS) {
      const int pos = j + rank_in_run(bs, bi, nB, nsc[j], nix[j], ld);
      if (pos < itopk) {
        ts[pos] = nsc[j];
        ti[pos] = nix[j];
        te[pos] = 0;
      }
    }
    nB = min(itopk, nB + nn);
    nv += nn;
    swap_ptr(bs, ts);
    swap_ptr(bi, ti);
    swap_ptr(be, te);
    __syncthreads();
    if (it == max_iter) break;

    // the parents: the first `width` unexpanded entries of B
    int np = 0;
    for (int b0 = 0; b0 < nB && np < width; b0 += GS_THREADS) {
      const int i = b0 + threadIdx.x;
      const int f = i < nB && !be[i];
      int tot;
      const int incl = block_scan(f, warp_sums, &tot);
      if (f && np + incl <= width) par[np + incl - 1] = i;
      np += tot;
    }
    np = min(np, width);
    __syncthreads();
    if (np == 0) break;
    ++it;

    // N_t: the parents' entries not in V, in (parent, edge) order, each row once
    const int ns = np * degree;
    for (int s = threadIdx.x; s < ns; s += GS_THREADS) {
      const int a = s / degree;
      const int c = graph[bi[par[a]] * degree + (s - a * degree)];
      cand[s] = c >= 0 && !gs_lookup(H, mask, l.log2S, c) ? c : -1;
    }
    __syncthreads();
    for (int s = threadIdx.x; s < ns; s += GS_THREADS)
      if (cand[s] >= 0) first_slot_note(F, fmask, l.log2F, cand[s], s);
    for (int a = threadIdx.x; a < np; a += GS_THREADS) be[par[a]] = 1;
    __syncthreads();
    nn = 0;
    for (int s0 = 0; s0 < ns; s0 += GS_THREADS) {
      const int s = s0 + threadIdx.x;
      const int c = s < ns ? cand[s] : -1;
      const bool keep = c >= 0 && first_slot(F, fmask, l.log2F, c) == s;
      int tot;
      const int incl = block_scan(static_cast<int>(keep), warp_sums, &tot);
      if (keep) {
        nix[nn + incl - 1] = c;
        gs_insert(H, mask, l.log2S, c);
      }
      nn += tot;
    }
    __syncthreads();
    for (uint32_t h = threadIdx.x; h <= fmask; h += GS_THREADS) F[h] = GS_FREE;
  }
  for (int t = threadIdx.x; t < k; t += GS_THREADS) {
    out_s[qi * k + t] = t < nB ? bs[t] : -INFINITY;
    out_i[qi * k + t] = t < nB ? bi[t] : -1;
  }
  if (threadIdx.x == 0) {
    n_vis[qi] = static_cast<int>(nv);
    n_iter[qi] = it;
  }
}

}  // namespace
}  // namespace dirb

using namespace dirb;

extern "C" {

int dirb200_graph_prune(const int* knn_dev, int64_t n, int K, int degree, int* fwd_dev, void* stream_) {
  DIRB_REQUIRE(n >= 1 && n < (int64_t(1) << 31) && K >= 0 && degree >= 1 && fwd_dev && (K == 0 || knn_dev),
               DIRB200_EINVAL, "bad arguments");
  DIRB_REQUIRE(K <= GRAPH_MAX_K && degree <= GRAPH_MAX_DEGREE, DIRB200_ENOTSUP,
               "build_k %d / degree %d: at most %d / %d", K, degree, GRAPH_MAX_K, GRAPH_MAX_DEGREE);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  static std::atomic<uint64_t> once{0};
  if (first_launch_on_device(once))
    DIRB_CUDA(cudaFuncSetAttribute(graph_prune_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   static_cast<int>(prune_smem(GRAPH_MAX_K))));
  graph_prune_kernel<<<static_cast<unsigned>(n), PRUNE_THREADS, prune_smem(K), stream>>>(knn_dev, K, degree, fwd_dev);
  count_launch();
  DIRB_CUDA(cudaGetLastError());
  return 0;
}

int dirb200_graph_merge(const int* fwd_dev, int64_t n, int degree, const int64_t* rev_off_dev, const int* rev_src_dev,
                        int* graph_dev, void* stream_) {
  DIRB_REQUIRE(n >= 1 && n < (int64_t(1) << 31) && degree >= 1 && fwd_dev && rev_off_dev && graph_dev,
               DIRB200_EINVAL, "bad arguments");
  DIRB_REQUIRE(degree <= GRAPH_MAX_DEGREE, DIRB200_ENOTSUP, "degree %d: at most %d", degree, GRAPH_MAX_DEGREE);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  graph_merge_kernel<<<static_cast<unsigned>(ceil_div(n, MERGE_WARPS)), MERGE_WARPS * 32, 0, stream>>>(
      fwd_dev, n, degree, rev_off_dev, rev_src_dev, graph_dev);
  count_launch();
  DIRB_CUDA(cudaGetLastError());
  return 0;
}

size_t dirb200_graph_search_smem_bytes(int n_seeds, int itopk, int width, int degree, int max_iter) {
  if (n_seeds < 1 || itopk < 1 || width < 1 || degree < 1 || max_iter < 0) return 0;
  if (static_cast<int64_t>(width) * degree > (1 << 20) ||
      static_cast<int64_t>(max_iter) * width * degree + n_seeds > (int64_t(1) << 28))
    return SIZE_MAX;
  return gs_layout(n_seeds, itopk, width, degree, max_iter).total + GS_WARPS * sizeof(int);
}

int dirb200_graph_search(const float* q_dev, int Q, int D, const float* x_dev, int64_t n, const int* graph_dev,
                         int degree, const int* seeds_dev, int n_seeds, int itopk, int width, int max_iter, int k,
                         double* out_scores, int64_t* out_rows, int64_t* vis_rows, double* vis_scores, int* n_visited,
                         int* n_iter, void* stream_) {
  DIRB_REQUIRE(Q >= 1 && D > 0 && D % 4 == 0 && n >= 1 && n < (int64_t(1) << 31) && degree >= 1 && n_seeds >= 1 &&
                   n_seeds <= n && itopk >= 1 && width >= 1 && max_iter >= 0 && k >= 1 && k <= itopk && q_dev &&
                   x_dev && graph_dev && seeds_dev && out_scores && out_rows && n_visited && n_iter &&
                   (vis_rows == nullptr) == (vis_scores == nullptr),
               DIRB200_EINVAL, "bad arguments");
  const size_t smem = dirb200_graph_search_smem_bytes(n_seeds, itopk, width, degree, max_iter);
  int dev = 0, optin = 0;
  DIRB_CUDA(cudaGetDevice(&dev));
  DIRB_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  DIRB_REQUIRE(smem <= static_cast<size_t>(optin), DIRB200_EINVAL,
               "graph search needs %zu bytes of shared memory per query (n_seeds %d, itopk %d, width %d, degree %d, "
               "max_iter %d); the device has %d", smem, n_seeds, itopk, width, degree, max_iter, optin);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  static std::atomic<uint64_t> once{0};
  if (first_launch_on_device(once))
    DIRB_CUDA(cudaFuncSetAttribute(graph_search_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   optin - static_cast<int>(GS_WARPS * sizeof(int))));   // less the static warp sums
  const int64_t vcap = static_cast<int64_t>(n_seeds) + static_cast<int64_t>(max_iter) * width * degree;
  graph_search_kernel<<<static_cast<unsigned>(Q), GS_THREADS, smem - GS_WARPS * sizeof(int), stream>>>(
      q_dev, D, x_dev, graph_dev, degree, seeds_dev, n_seeds, itopk, width, max_iter, k, out_scores, out_rows, vis_rows,
      vis_scores, vcap, n_visited, n_iter);
  count_launch();
  DIRB_CUDA(cudaGetLastError());
  return 0;
}

}  // extern "C"
