// Threshold counts for label-based AP (dirb200_index_count_ge): the kernels live in label_count.cu, the entry point
// in search.cu (which owns the index handle and its workspace).
#pragma once
#include "common.h"

namespace dirb {

struct CountGeArgs {
  const float* q32 = nullptr;        // [Q][D] queries
  int Q = 0;
  const float* db32 = nullptr;       // [N][D] rows of this shard
  int64_t N = 0, offset = 0;         // global index of row r = r + offset
  int D = 0;
  const int* thr_off = nullptr;      // [Q+1] CSR offsets of the thresholds (device)
  const float* thr = nullptr;        // [T] thresholds, descending within each query
  int T = 0;
  const int64_t* skip_row = nullptr; // [Q] global row not counted for query q (-1: none), or nullptr
  int64_t* count = nullptr;          // [T] out: rows of this shard with fl32(score) >= thr[t]
  double eps = 0;                    // > 0: absolute bound on |fp64 tensor-core score - exact score|; 0: from the norms
  int band_cap = 0;                  // capacity of the band list (entries)
};

struct CountGeStats {
  int64_t band = 0;                  // (query, row) pairs re-scored exactly because they fell within eps of a boundary
  int64_t fallback = 0;              // queries counted exactly over all rows after a band-list overflow
};

size_t count_ge_ws_bytes(int Q, int T, int band_cap);
// Enqueues everything on `stream` and synchronises it once (the list of overflowed queries goes to the host).
int count_ge_run(const CountGeArgs& a, void* ws, CountGeStats* st, cudaStream_t stream);

}  // namespace dirb
