// Connected components of a self-join's pair graph and its duplicate groups (DESIGN.md section 4.8, rule J4).
//
//   cc_hook_kernel       one thread per pair (i, j): the roots of i and j; when they differ the larger root is hooked
//                        to the smaller with atomicMin.  A parent is always smaller than its node and in its component,
//                        whatever order the atomics take.
//   cc_compress_kernel   every node points at its root (pointer jumping).
// The two alternate until no pair joins two roots; the root of a component is then its smallest row, so the labels
// are rule J4's on every run.
//   groups               component sizes (counts), the rows of components of >= 2 rows ordered by (label, row) with
//                        sort_runs_merge (key -label, then row), and the group offsets from one block-wide scan.
#include <limits.h>

#include <algorithm>

#include "block.cuh"
#include "common.h"

namespace dirb {
namespace {

constexpr int CC_THREADS = 256;
constexpr int SCAN_THREADS = 1024;

__global__ void cc_init_kernel(int64_t* __restrict__ parent, int64_t n) {
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    parent[i] = i;
}

__device__ __forceinline__ int64_t cc_root(const volatile int64_t* parent, int64_t x) {
  for (;;) {
    const int64_t p = parent[x];
    if (p == x) return x;
    x = p;
  }
}

__global__ void cc_hook_kernel(const int64_t* __restrict__ row_ptr, const int64_t* __restrict__ col, int64_t n,
                               int64_t nnz, int64_t* parent, int* __restrict__ changed) {
  for (int64_t e = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; e < nnz;
       e += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    int64_t lo = 0, hi = n;                       // the row of pair e: last i with row_ptr[i] <= e
    while (hi - lo > 1) {
      const int64_t mid = (lo + hi) >> 1;
      if (__ldg(row_ptr + mid) <= e) lo = mid; else hi = mid;
    }
    const int64_t ri = cc_root(parent, lo), rj = cc_root(parent, __ldg(col + e));
    if (ri != rj) {
      atomicMin(reinterpret_cast<long long*>(parent + max(ri, rj)), static_cast<long long>(min(ri, rj)));
      *changed = 1;
    }
  }
}

__global__ void cc_compress_kernel(int64_t* parent, int64_t n) {
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    parent[i] = cc_root(parent, i);
}

__global__ void group_size_kernel(const int64_t* __restrict__ label, int64_t n, int* __restrict__ size) {
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    atomicAdd(size + label[i], 1);
}

// Rows of components with >= 2 rows, in any order (the sort fixes it): key -label, so (key desc, row asc) is
// (label asc, row asc).
__global__ void group_gather_kernel(const int64_t* __restrict__ label, int64_t n, const int* __restrict__ size,
                                    int* __restrict__ rows, double* __restrict__ key, int* __restrict__ cnt) {
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t l = label[i];
    if (size[l] >= 2) {
      const int pos = atomicAdd(cnt, 1);
      rows[pos] = static_cast<int>(i);
      key[pos] = -static_cast<double>(l);
    }
  }
}

// One block: position p of the ordered members starts a group when its label differs from the previous member's;
// group g's offset is the p of its g-th start.  counts[0] = groups, counts[1] = members.
__global__ void __launch_bounds__(SCAN_THREADS) group_offsets_kernel(const int64_t* __restrict__ members,
                                                                     const int64_t* __restrict__ label, int m,
                                                                     int64_t* __restrict__ group_off,
                                                                     int64_t* __restrict__ counts) {
  __shared__ int warp_sums[SCAN_THREADS / 32];
  int64_t carry = 0;
  for (int base = 0; base < m; base += SCAN_THREADS) {
    const int p = base + threadIdx.x;
    const int start = (p < m && (p == 0 || label[members[p]] != label[members[p - 1]])) ? 1 : 0;
    int tot;
    const int incl = block_scan(start, warp_sums, &tot);
    if (start) group_off[carry + incl - 1] = p;
    carry += tot;
  }
  if (threadIdx.x == 0) {
    group_off[carry] = m;
    counts[0] = carry;
    counts[1] = m;
  }
}

struct GroupWs {
  int* size;
  SortScratch sort;
  double* out_key;
  int* cnt;
  int64_t* counts;
  unsigned long long* status;
  size_t total;
};
GroupWs group_ws(void* base, int64_t n) {
  Carver c(base);
  GroupWs w;
  w.size = c.take<int>(n);
  w.sort = take_sort_scratch(c, 1, sort_run_cap(std::max<int64_t>(n, 1)));
  w.out_key = c.take<double>(n);
  w.cnt = c.take<int>(1);
  w.counts = c.take<int64_t>(2);
  w.status = c.take<unsigned long long>(8);
  w.total = c.used;
  return w;
}

unsigned grid_for(int64_t n) { return static_cast<unsigned>(std::max<int64_t>(1, std::min<int64_t>(ceil_div(n, CC_THREADS), 8192))); }

}  // namespace
}  // namespace dirb

using namespace dirb;

extern "C" {

size_t dirb200_join_components_workspace_bytes(int64_t n) {
  (void)n;
  return 256;
}

int dirb200_join_components(const int64_t* row_ptr_dev, const int64_t* col_dev, int64_t n, int64_t nnz, void* ws_dev,
                            int64_t* labels_dev, void* stream_) {
  DIRB_REQUIRE(n >= 1 && nnz >= 0 && labels_dev && ws_dev && (nnz == 0 || (row_ptr_dev && col_dev)), DIRB200_EINVAL,
               "bad arguments");
  DIRB_REQUIRE(n < (int64_t(1) << 31), DIRB200_ENOTSUP, "too many rows (%lld)", static_cast<long long>(n));
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int* changed = static_cast<int*>(ws_dev);
  cc_init_kernel<<<grid_for(n), CC_THREADS, 0, stream>>>(labels_dev, n);
  count_launch();
  if (nnz > 0) {
    for (;;) {
      int flag = 0;
      DIRB_CUDA(cudaMemsetAsync(changed, 0, 4, stream));
      cc_hook_kernel<<<grid_for(nnz), CC_THREADS, 0, stream>>>(row_ptr_dev, col_dev, n, nnz, labels_dev, changed);
      cc_compress_kernel<<<grid_for(n), CC_THREADS, 0, stream>>>(labels_dev, n);
      count_launch(2);
      DIRB_CUDA(cudaMemcpyAsync(&flag, changed, 4, cudaMemcpyDeviceToHost, stream));
      DIRB_CUDA(cudaStreamSynchronize(stream));
      if (!flag) break;
    }
  }
  DIRB_CUDA(cudaGetLastError());
  return 0;
}

size_t dirb200_join_groups_workspace_bytes(int64_t n) {
  if (n < 1) return 0;
  return group_ws(nullptr, n).total;
}

int dirb200_join_groups(const int64_t* labels_dev, int64_t n, void* ws_dev, int64_t* group_off_dev, int64_t* members_dev,
                        int64_t counts_out[2], void* stream_) {
  DIRB_REQUIRE(n >= 1 && labels_dev && ws_dev && group_off_dev && members_dev && counts_out, DIRB200_EINVAL,
               "bad arguments");
  DIRB_REQUIRE(n < (int64_t(1) << 31), DIRB200_ENOTSUP, "too many rows (%lld)", static_cast<long long>(n));
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const GroupWs w = group_ws(ws_dev, n);
  DIRB_CUDA(cudaMemsetAsync(w.size, 0, static_cast<size_t>(n) * 4, stream));
  DIRB_CUDA(cudaMemsetAsync(w.cnt, 0, 4, stream));
  group_size_kernel<<<grid_for(n), CC_THREADS, 0, stream>>>(labels_dev, n, w.size);
  group_gather_kernel<<<grid_for(n), CC_THREADS, 0, stream>>>(labels_dev, n, w.size, w.sort.rows, w.sort.sc, w.cnt);
  count_launch(2);
  int m = 0;
  DIRB_CUDA(cudaMemcpyAsync(&m, w.cnt, 4, cudaMemcpyDeviceToHost, stream));
  DIRB_CUDA(cudaStreamSynchronize(stream));
  if (m > 0) {
    DIRB_TRY(sort_runs_merge(w.sort.rows, w.cnt, sort_run_cap(m), w.sort.sc, w.sort.run_ix, 1, m, 0, w.status, w.out_key,
                             members_dev, stream));
  }
  group_offsets_kernel<<<1, SCAN_THREADS, 0, stream>>>(members_dev, labels_dev, m, group_off_dev, w.counts);
  count_launch();
  DIRB_CUDA(cudaMemcpyAsync(counts_out, w.counts, 16, cudaMemcpyDeviceToHost, stream));
  DIRB_CUDA(cudaStreamSynchronize(stream));
  DIRB_CUDA(cudaGetLastError());
  return 0;
}

}  // extern "C"
