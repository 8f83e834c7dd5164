// Test-only wrappers around the block primitives of block.cuh, one small kernel per primitive, each with an extern "C"
// launcher that returns the cudaError_t of its launch.  Built by build_ext.py into libdirb200_blocktest.so, which is not
// part of the library; tests/test_gpu_block.py compares every result with the numpy model of tests/block_model.py.
// Nothing here restates a caller: each kernel loads its inputs, calls the header and stores what it returned.
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "../deep-image-retrieval_b200/csrc/block.cuh"

namespace {
using namespace dirb;

// The orders the callers sort by.
struct ResultOrder {                     // search finish, deep run sort (int index), graph search (int64_t index)
  template <class I>
  __device__ bool operator()(double sa, I ia, double sb, I ib) const { return ranks_before(sa, ia, sb, ib); }
};
struct ByIndex {                         // diffusion's neighbour sort: (index, weight) by index
  __device__ bool operator()(int a, double, int b, double) const { return a < b; }
};
struct Ascending {                       // keys only: trunc_build (uint64_t), graph_prune (uint32_t)
  template <class K>
  __device__ bool operator()(K a, K b) const { return a < b; }
};

template <class K>
__host__ __device__ size_t val_offset(int P) { return (static_cast<size_t>(P) * sizeof(K) + 15) & ~static_cast<size_t>(15); }

// Block b sorts its P entries key[b * P ..], val[b * P ..] (V = void: keys only), in place in global memory or through
// dynamic shared memory.  Straight after the call, with no barrier of its own, entry j of seen_* takes entry
// (7 j + 3) mod P, which another thread wrote: the sort's closing barrier is what makes that read safe.
template <int NT, class K, class V, class Before>
__global__ void __launch_bounds__(NT, 1) sort_kernel(K* gkey, std::conditional_t<std::is_void_v<V>, char, V>* gval,
                                                     int P, int in_smem, K* seen_key,
                                                     std::conditional_t<std::is_void_v<V>, char, V>* seen_val) {
  using VS = std::conditional_t<std::is_void_v<V>, char, V>;
  extern __shared__ __align__(16) unsigned char sm[];
  const int64_t o = static_cast<int64_t>(blockIdx.x) * P;
  K* key = gkey + o;
  VS* val = std::is_void_v<V> ? nullptr : gval + o;
  if (in_smem) {
    K* sk = reinterpret_cast<K*>(sm);
    VS* sv = reinterpret_cast<VS*>(sm + val_offset<K>(P));
    for (int j = threadIdx.x; j < P; j += NT) {
      sk[j] = key[j];
      if constexpr (!std::is_void_v<V>) sv[j] = val[j];
    }
    key = sk;
    val = sv;
  }
  __syncthreads();
  if constexpr (std::is_void_v<V>) block_bitonic_sort<NT>(key, P, Before{});
  else block_bitonic_sort<NT>(key, val, P, Before{});
  for (int j = threadIdx.x; j < P; j += NT) {
    const int src = (7 * j + 3) & (P - 1);
    seen_key[o + j] = key[src];
    if constexpr (!std::is_void_v<V>) seen_val[o + j] = val[src];
  }
  __syncthreads();
  if (in_smem)
    for (int j = threadIdx.x; j < P; j += NT) {
      gkey[o + j] = key[j];
      if constexpr (!std::is_void_v<V>) gval[o + j] = val[j];
    }
}

template <int NT, class K, class V, class Before, class VS>
int sort_at(K* key, VS* val, int P, int blocks, int in_smem, K* seen_key, VS* seen_val) {
  const auto kern = sort_kernel<NT, K, V, Before>;
  const size_t smem = in_smem ? val_offset<K>(P) + (std::is_void_v<V> ? 0 : static_cast<size_t>(P) * sizeof(VS)) : 0;
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
  if (e != cudaSuccess) return e;
  kern<<<blocks, NT, smem>>>(key, val, P, in_smem, seen_key, seen_val);
  return cudaGetLastError();
}

// P a power of two; nt one of the block sizes below.
template <class K, class V, class Before, class VS>
int sort_nt(int nt, K* key, VS* val, int P, int blocks, int in_smem, K* seen_key, VS* seen_val) {
  if (P < 1 || (P & (P - 1)) != 0 || blocks < 1) return cudaErrorInvalidValue;
  switch (nt) {
    case 32: return sort_at<32, K, V, Before>(key, val, P, blocks, in_smem, seen_key, seen_val);
    case 128: return sort_at<128, K, V, Before>(key, val, P, blocks, in_smem, seen_key, seen_val);
    case 256: return sort_at<256, K, V, Before>(key, val, P, blocks, in_smem, seen_key, seen_val);
    case 512: return sort_at<512, K, V, Before>(key, val, P, blocks, in_smem, seen_key, seen_val);
    case 1024: return sort_at<1024, K, V, Before>(key, val, P, blocks, in_smem, seen_key, seen_val);
    default: return cudaErrorInvalidValue;
  }
}

// Block b runs three block_scans back to back on one warp_sums, over in[b][c][t] for c = 0, 1, 2; thread t stores its
// inclusive sum and the total it was given.
template <class T>
__global__ void __launch_bounds__(1024) scan_kernel(const T* in, T* incl, T* total) {
  __shared__ T warp_sums[32];
  const int64_t o = static_cast<int64_t>(blockIdx.x) * 3 * blockDim.x + threadIdx.x, s = blockDim.x;
  const T a = in[o], b = in[o + s], c = in[o + 2 * s];
  T ta, tb, tc;
  const T ia = block_scan(a, warp_sums, &ta);
  const T ib = block_scan(b, warp_sums, &tb);
  const T ic = block_scan(c, warp_sums, &tc);
  incl[o] = ia, incl[o + s] = ib, incl[o + 2 * s] = ic;
  total[o] = ta, total[o + s] = tb, total[o + 2 * s] = tc;
}

template <class T>
int scan_launch(int nt, const T* in, T* incl, T* total, int blocks) {
  if (nt < 32 || nt > 1024 || nt % 32 != 0 || blocks < 1) return cudaErrorInvalidValue;
  scan_kernel<T><<<blocks, nt>>>(in, incl, total);
  return cudaGetLastError();
}

template <class T>
__global__ void warp_scan_kernel(const T* in, T* out, int64_t n) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) out[i] = warp_scan(in[i]);                  // n a multiple of 32: whole warps only
}

template <class T>
int warp_scan_launch(const T* in, T* out, int64_t n) {
  if (n < 32 || n % 32 != 0) return cudaErrorInvalidValue;
  warp_scan_kernel<T><<<static_cast<unsigned>((n + 255) / 256), 256>>>(in, out, n);
  return cudaGetLastError();
}

// Block b selects the k1[b]-th and then, sharing hist / bc, the k2[b]-th largest key: out[2b], out[2b + 1].
template <class Key, class Int, class KeyOf>
__global__ void __launch_bounds__(1024) kth_kernel(KeyOf key_of, Int n, const int* k1, const int* k2, Key* out) {
  __shared__ uint32_t hist[256], bc[2];
  const Key a = block_radix_kth<Key>(key_of, n, k1[blockIdx.x], hist, bc);
  const Key b = block_radix_kth<Key>(key_of, n, k2[blockIdx.x], hist, bc);
  if (threadIdx.x == 0) out[2 * blockIdx.x] = a, out[2 * blockIdx.x + 1] = b;
}

template <class Key, class Int>
struct KeyLoad {
  const Key* p;
  __device__ Key operator()(Int i) const { return p[i]; }
};
struct FloatKeyLoad {                    // the search's form: keys are f2key of fp32 scores
  const float* p;
  __device__ uint32_t operator()(int i) const { return f2key(p[i]); }
};

template <class Key, class Int, class KeyOf>
int kth_launch(int nt, KeyOf key_of, Int n, const int* k1, const int* k2, int blocks, Key* out) {
  if (nt < 32 || nt > 1024 || nt % 32 != 0 || n < 1 || blocks < 1) return cudaErrorInvalidValue;
  kth_kernel<Key, Int><<<blocks, nt>>>(key_of, n, k1, k2, out);
  return cudaGetLastError();
}

template <class Load>
__global__ void rank_kernel(const double* sc, const int64_t* ix, int n, const double* ps, const int64_t* pi, int np,
                            int* out, Load load) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < np) out[t] = rank_in_run(sc, ix, n, ps[t], pi[t], load);
}
struct PlainLoad {                       // merge_lists, graph search
  template <class T>
  __device__ T operator()(const T* p) const { return *p; }
};
struct CgLoad {                          // merge_runs
  template <class T>
  __device__ T operator()(const T* p) const { return __ldcg(p); }
};

// Keys [base, base + count) with count <= 2^31: bad[0] counts f2key(key2f(k)) != k, bad[1] counts keys k whose float
// does not lie below that of k + 1 (NaNs skipped; -0 at k = 0x7fffffff and +0 above it is the one allowed tie).
__global__ void key_sweep_kernel(uint32_t base, uint32_t count, unsigned long long* bad) {
  unsigned long long round = 0, order = 0;
  for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < count; t += gridDim.x * blockDim.x) {
    const uint32_t k = base + t;
    const float f = key2f(k);
    round += f2key(f) != k;
    if (k != 0xffffffffu) {
      const float g = key2f(k + 1);
      if (!isnan(f) && !isnan(g) && !(f < g))
        order += !(k == 0x7fffffffu && __float_as_uint(f) == 0x80000000u && __float_as_uint(g) == 0u);
    }
  }
  if (round) atomicAdd(bad, round);
  if (order) atomicAdd(bad + 1, order);
}

__global__ void elementwise_kernel(const float* f, uint32_t* f2k, const uint32_t* k, float* k2f, const double* sa,
                                   const int64_t* ia, const double* sb, const int64_t* ib, uint64_t* fk, uint8_t* before,
                                   uint8_t* before_key, int n) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  f2k[t] = f2key(f[t]);
  k2f[t] = key2f(k[t]);
  fk[t] = fkey(sa[t]);
  before[t] = ranks_before(sa[t], ia[t], sb[t], ib[t]);
  before_key[t] = ranks_before(fkey(sa[t]), ia[t], fkey(sb[t]), ib[t]);
}

unsigned grid_of(int64_t n) { return static_cast<unsigned>((n + 255) / 256); }
}  // namespace

extern "C" {
// block_bitonic_sort: `blocks` independent arrays of P entries; in_smem != 0 sorts them in dynamic shared memory.
int dirb_blocktest_sort_f64_i32(int nt, double* s, int* i, int P, int blocks, int in_smem, double* ss, int* si) {
  return sort_nt<double, int, ResultOrder>(nt, s, i, P, blocks, in_smem, ss, si);
}
int dirb_blocktest_sort_f64_i64(int nt, double* s, int64_t* i, int P, int blocks, int in_smem, double* ss, int64_t* si) {
  return sort_nt<double, int64_t, ResultOrder>(nt, s, i, P, blocks, in_smem, ss, si);
}
int dirb_blocktest_sort_i32_f64(int nt, int* i, double* w, int P, int blocks, int in_smem, int* si, double* sw) {
  return sort_nt<int, double, ByIndex>(nt, i, w, P, blocks, in_smem, si, sw);
}
int dirb_blocktest_sort_u64(int nt, uint64_t* k, int P, int blocks, int in_smem, uint64_t* sk) {
  return sort_nt<uint64_t, void, Ascending, char>(nt, k, nullptr, P, blocks, in_smem, sk, nullptr);
}
int dirb_blocktest_sort_u32(int nt, uint32_t* k, int P, int blocks, int in_smem, uint32_t* sk) {
  return sort_nt<uint32_t, void, Ascending, char>(nt, k, nullptr, P, blocks, in_smem, sk, nullptr);
}

// block_scan: in / incl / total are [blocks][3][nt].
int dirb_blocktest_scan_i32(int nt, const int* in, int* incl, int* total, int blocks) {
  return scan_launch(nt, in, incl, total, blocks);
}
int dirb_blocktest_scan_i64(int nt, const long long* in, long long* incl, long long* total, int blocks) {
  return scan_launch(nt, in, incl, total, blocks);
}
int dirb_blocktest_scan_u64(int nt, const unsigned long long* in, unsigned long long* incl, unsigned long long* total,
                            int blocks) {
  return scan_launch(nt, in, incl, total, blocks);
}
int dirb_blocktest_warp_scan_i32(const int* in, int* out, int64_t n) { return warp_scan_launch(in, out, n); }
int dirb_blocktest_warp_scan_i64(const long long* in, long long* out, int64_t n) { return warp_scan_launch(in, out, n); }
int dirb_blocktest_warp_scan_u64(const unsigned long long* in, unsigned long long* out, int64_t n) {
  return warp_scan_launch(in, out, n);
}

// block_radix_kth: one block per (k1[b], k2[b]) pair over the same n keys, 1 <= k <= n.
int dirb_blocktest_kth_u32(int nt, const uint32_t* key, int n, const int* k1, const int* k2, int blocks, uint32_t* out) {
  return kth_launch<uint32_t, int>(nt, KeyLoad<uint32_t, int>{key}, n, k1, k2, blocks, out);
}
int dirb_blocktest_kth_u32_n64(int nt, const uint32_t* key, int64_t n, const int* k1, const int* k2, int blocks,
                               uint32_t* out) {
  return kth_launch<uint32_t, int64_t>(nt, KeyLoad<uint32_t, int64_t>{key}, n, k1, k2, blocks, out);
}
int dirb_blocktest_kth_u64(int nt, const uint64_t* key, int64_t n, const int* k1, const int* k2, int blocks, uint64_t* out) {
  return kth_launch<uint64_t, int64_t>(nt, KeyLoad<uint64_t, int64_t>{key}, n, k1, k2, blocks, out);
}
int dirb_blocktest_kth_f32(int nt, const float* x, int n, const int* k1, const int* k2, int blocks, uint32_t* out) {
  return kth_launch<uint32_t, int>(nt, FloatKeyLoad{x}, n, k1, k2, blocks, out);
}

// rank_in_run of each probe (ps[t], pi[t]) in the run (sc, ix)[0 .. n), through plain loads or __ldcg.
int dirb_blocktest_rank(const double* sc, const int64_t* ix, int n, const double* ps, const int64_t* pi, int np, int ldcg,
                        int* out) {
  if (np < 1) return cudaErrorInvalidValue;
  if (ldcg) rank_kernel<<<grid_of(np), 256>>>(sc, ix, n, ps, pi, np, out, CgLoad{});
  else rank_kernel<<<grid_of(np), 256>>>(sc, ix, n, ps, pi, np, out, PlainLoad{});
  return cudaGetLastError();
}

int dirb_blocktest_key_sweep(uint32_t base, uint32_t count, unsigned long long* bad) {
  if (count == 0 || count > 0x80000000u) return cudaErrorInvalidValue;
  key_sweep_kernel<<<4096, 256>>>(base, count, bad);
  return cudaGetLastError();
}

// f2key, key2f, fkey and both ranks_before overloads, element by element.
int dirb_blocktest_elementwise(const float* f, uint32_t* f2k, const uint32_t* k, float* k2f, const double* sa,
                               const int64_t* ia, const double* sb, const int64_t* ib, uint64_t* fk, uint8_t* before,
                               uint8_t* before_key, int n) {
  if (n < 1) return cudaErrorInvalidValue;
  elementwise_kernel<<<grid_of(n), 256>>>(f, f2k, k, k2f, sa, ia, sb, ib, fk, before, before_key, n);
  return cudaGetLastError();
}
}
