// Block-level primitives of the retrieval kernels: the result order, order-preserving keys, a bitonic sort, a scan, a
// radix select and the rank of an entry in a sorted run.
#pragma once

#include <stdint.h>

#include <type_traits>

namespace dirb {

// The library's result order: exact score descending, ties to the lower index, i.e. sa > sb || (sa == sb && ia < ib).
// -0 == +0, as doubles compare.  (Written as a branch: search_finish_kernel then compiles as it did before the sort was
// shared, in 32 registers.)
__device__ __forceinline__ bool ranks_before(double sa, int64_t ia, double sb, int64_t ib) {
  if (sa != sb) return sa > sb;
  return ia < ib;
}
// The same order on the keys of fkey.
__device__ __forceinline__ bool ranks_before(uint64_t ka, int64_t ia, uint64_t kb, int64_t ib) {
  if (ka != kb) return ka > kb;
  return ia < ib;
}

// Monotone increasing map float -> uint32 and back.  -0 maps just below +0.
__device__ __forceinline__ uint32_t f2key(float f) {
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key2f(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// Monotone map double -> uint64 with -0 and +0 the same key.
__device__ __forceinline__ uint64_t fkey(double v) {
  const uint64_t b = static_cast<uint64_t>(__double_as_longlong(v + 0.0));    // -0 + 0 = +0
  return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}

// Sorts the P entries (key, val) of shared or global memory, P a power of two, so that before(key[i], val[i], key[j],
// val[j]) holds for no i > j; with before(ka, kb) and val == nullptr (the keys-only form below) only the keys move.
// NT = blockDim.x.  Entries that compare equal both ways may end in either order, so their payloads must not matter
// (the callers' equal keys are padding).  Ends with a barrier.
template <int NT, class K, class V, class Before>
__device__ __forceinline__ void block_bitonic_sort(K* key, V* val, int P, Before before) {
  for (int size = 2; size <= P; size <<= 1)
    for (int st = size >> 1; st > 0; st >>= 1) {
      for (int i = threadIdx.x; i < P / 2; i += NT) {
        const int lo = 2 * i - (i & (st - 1)), hi = lo + st;
        const bool up = (lo & size) == 0;          // this block of the network sorts in `before` order
        const K ka = key[lo], kb = key[hi];
        if constexpr (std::is_void_v<V>) {
          if (before(ka, kb) != up) { key[lo] = kb; key[hi] = ka; }
        } else {
          const V va = val[lo], vb = val[hi];
          if (before(ka, va, kb, vb) != up) {
            key[lo] = kb; key[hi] = ka;
            val[lo] = vb; val[hi] = va;
          }
        }
      }
      __syncthreads();
    }
}
template <int NT, class K, class Before>
__device__ __forceinline__ void block_bitonic_sort(K* key, int P, Before before) {
  block_bitonic_sort<NT, K, void>(key, nullptr, P, before);
}

// Inclusive sum over the lanes of a warp.
template <class T>
__device__ __forceinline__ T warp_scan(T v) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T y = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += y;
  }
  return v;
}

// Inclusive sum of one value per thread over the block (blockDim.x a multiple of 32); *total = the block's sum.
// warp_sums: blockDim.x / 32 shared values.  Every thread must call it; it may be called again at once.
template <class T>
__device__ __forceinline__ T block_scan(T v, T* warp_sums, T* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const T incl = warp_scan(v);
  if (lane == 31) warp_sums[warp] = incl;
  __syncthreads();
  T before = 0, tot = 0;
  for (int w = 0; w < static_cast<int>(blockDim.x >> 5); ++w) {
    if (w < warp) before += warp_sums[w];
    tot += warp_sums[w];
  }
  __syncthreads();
  *total = tot;
  return incl + before;
}

// The k-th largest of the n keys key_of(0 .. n-1), 1 <= k <= n: block-wide MSB-first radix select, 8 bits per pass.
// Key is uint32_t or uint64_t.  Every thread must call it and gets the key.
template <class Key, class KeyOf, class Int>
__device__ Key block_radix_kth(KeyOf key_of, Int n, int k, uint32_t* hist /*[256]*/, uint32_t* bc /*[2]*/) {
  Key prefix = 0, mask = 0;
  int kk = k;
  for (int shift = 8 * (sizeof(Key) - 1); shift >= 0; shift -= 8) {
    for (int i = threadIdx.x; i < 256; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    // similarity scores share their high bits, so most keys of a pass land in one or two bins: aggregate the
    // lanes of a warp that hit the same bin and let one of them add the whole group
    const Int n_round = (n + 31) & ~static_cast<Int>(31);
    for (Int i = threadIdx.x; i < n_round; i += blockDim.x) {
      uint32_t bin = 0xffffffffu;
      if (i < n) {
        const Key key = key_of(i);
        if ((key & mask) == prefix) bin = static_cast<uint32_t>(key >> shift) & 255u;
      }
      const uint32_t peers = __match_any_sync(0xffffffffu, bin);
      if (bin != 0xffffffffu && (threadIdx.x & 31) == (__ffs(peers) - 1)) atomicAdd(&hist[bin], static_cast<uint32_t>(__popc(peers)));
    }
    __syncthreads();
    if (threadIdx.x < 32) {
      // Find the bin holding the kk-th largest key: lane l owns bins [8l, 8l+8); a suffix scan over the lanes gives
      // the number of keys in higher bins, the owning lane walks its 8 bins.  (A single thread walking 256 bins
      // serially cost ~10 us per pass.)
      const int lane = threadIdx.x;
      uint32_t loc[8], sum = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        loc[j] = hist[8 * lane + j];
        sum += loc[j];
      }
      uint32_t suf = sum;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t v = __shfl_down_sync(0xffffffffu, suf, o);
        if (lane + o < 32) suf += v;
      }
      const uint32_t above = suf - sum;
      const uint32_t want = static_cast<uint32_t>(kk);
      if (above < want && want <= above + sum) {
        uint32_t cum = above;
#pragma unroll
        for (int j = 7; j >= 0; --j) {
          if (cum + loc[j] >= want) {
            bc[0] = 8 * lane + j;
            bc[1] = want - cum;
            break;
          }
          cum += loc[j];
        }
      }
    }
    __syncthreads();
    prefix |= static_cast<Key>(bc[0]) << shift;
    mask |= static_cast<Key>(255u) << shift;
    kk = bc[1];
    __syncthreads();
  }
  return prefix;
}

// The number of entries of a run ordered by ranks_before (empty entries, index < 0, only at its tail) that rank before
// (s, i), by binary search over its first n entries.  load(p) reads one element: a plain read, or __ldcg for a run
// another block wrote.
template <class Load>
__device__ __forceinline__ int rank_in_run(const double* sc, const int64_t* ix, int n, double s, int64_t i, Load load) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    const int64_t im = load(ix + mid);
    const double sm = load(sc + mid);
    if (im >= 0 && ranks_before(sm, im, s, i)) lo = mid + 1; else hi = mid;
  }
  return lo;
}

}  // namespace dirb
