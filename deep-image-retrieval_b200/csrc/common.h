// Host-side plumbing shared by all translation units: error reporting, status codes, TMA descriptor encoding.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>

#include "../../include/dirb200.h"

namespace dirb {

void set_error(const char* fmt, ...);
const char* last_error();

#define DIRB_CUDA(expr)                                                                         \
  do {                                                                                          \
    cudaError_t _e = (expr);                                                                    \
    if (_e != cudaSuccess) {                                                                    \
      ::dirb::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return static_cast<int>(_e);                                                              \
    }                                                                                           \
  } while (0)

#define DIRB_REQUIRE(cond, code, ...)   \
  do {                                  \
    if (!(cond)) {                      \
      ::dirb::set_error(__VA_ARGS__);   \
      return (code);                    \
    }                                   \
  } while (0)

#define DIRB_TRY(expr)         \
  do {                         \
    int _s = (expr);           \
    if (_s != 0) return _s;    \
  } while (0)

inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

// Typed sub-buffers of one workspace, handed out in order; each piece is rounded up to `align` bytes, so `used` is the
// sum of the rounded pieces.  With a null base the pointers are null and only `used` counts: a layout function
// X_ws(void* base, ...) gives both the buffer's size (base = nullptr) and its pointers.
struct Carver {
  char* base;
  size_t align, used = 0;
  explicit Carver(void* b, size_t a = 256) : base(static_cast<char*>(b)), align(a) {}
  template <typename T>
  T* take(size_t n) {
    T* p = base ? reinterpret_cast<T*>(base + used) : nullptr;
    used += (n * sizeof(T) + align - 1) / align * align;
    return p;
  }
};

// Grow the device buffer *p of *cap bytes to `need` bytes (contents are not kept; no-op when it is large enough).
// Pointer and capacity are cleared before the allocation and the capacity is set only once it succeeded, so after a
// failed call the buffer is empty rather than a null pointer with a stale capacity.
int grow_device(void** p, size_t* cap, size_t need);

// fp16 row-major [outer][inner] matrix, box = box_inner x box_outer elements, 128-byte swizzle.
int encode_tmap_2d(CUtensorMap* m, const void* base, uint64_t inner, uint64_t outer, uint64_t row_stride_bytes,
                   uint32_t box_inner, uint32_t box_outer);
// fp16 NHWC activation viewed as (C, W, H, B); box (64, tw*es, th*es, nb) traversed with element stride es
// on W and H (es = conv stride), 128-byte swizzle, out-of-bounds elements read as zero.
int encode_tmap_nhwc(CUtensorMap* m, const void* base, int B, int H, int W, int C, int tw, int th, int nb, int es);
// Input patch of a 3x3 / stride-1 / pad-1 convolution over an 8 x 16 output tile: HALO_W x HALO_H pixels of one image,
// 64 channels, no swizzle, stored channel-chunk-major in shared memory: [8 chunks of 8 channels][HALO_H][HALO_W][8]
// (16 bytes per pixel and chunk), the layout of K-major core matrices that wgmma reads without swizzle.  Coordinates
// (0, w, h, n, c/8); out-of-bounds pixels (the zero padding) read as zero.
constexpr int HALO_W = 10, HALO_H = 18;
int encode_tmap_nhwc_halo(CUtensorMap* m, const void* base, int B, int H, int W, int C);

// Launch `kern` with programmatic stream serialization (PDL): its CTAs may start while the previous kernel of the
// stream drains; the kernel must call pdl_wait() before touching data produced by its predecessor.
extern int g_use_pdl;
template <typename Kern, typename... Args>
inline cudaError_t launch_pdl(Kern kern, dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = g_use_pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, args...);
}

// cudaFuncSetAttribute is per (function, device) and costs ~1-2 us of host time: do it once per device, not per launch.
// `mask` is a function-local static of the launcher template instantiation.
inline bool first_launch_on_device(std::atomic<uint64_t>& mask) {
  int dev = 0;
  cudaGetDevice(&dev);
  const uint64_t bit = 1ull << (dev & 63);
  if (mask.load(std::memory_order_relaxed) & bit) return false;
  mask.fetch_or(bit, std::memory_order_relaxed);
  return true;
}

// dirb200_device_check of the current device: DIRB200_ENODEVICE when there is none or it is not sm_90.
int require_sm90();

// Sorted top-k of Q candidate lists (search.cu, the deep search's finish): list q holds min(cnt[q], cap2) pairs
// (rows[q * cap2 + i], sc[q * cap2 + i]), cap2 = sort_run_cap(longest list).  Runs of SORT_RUN are sorted in shared
// memory by (score desc, row asc) into sc / run_ix (the same layout), then merged by rank into out_score / out_idx
// [Q][k] (row + row_offset; (-inf, -1) past the end of a short list).  Q <= 65535.
constexpr int SORT_RUN = 2048;
inline int sort_run_cap(int64_t n) { return static_cast<int>(ceil_div(n, SORT_RUN) * SORT_RUN); }
struct SortScratch {
  int* rows;
  double* sc;
  int64_t* run_ix;
};
inline SortScratch take_sort_scratch(Carver& c, int64_t Q, int cap2) {
  const size_t n = static_cast<size_t>(Q) * cap2;
  return {c.take<int>(n), c.take<double>(n), c.take<int64_t>(n)};
}
int sort_runs_merge(const int* rows, const int* cnt, int cap2, double* sc, int64_t* run_ix, int Q, int k,
                    int64_t row_offset, unsigned long long* status, double* out_score, int64_t* out_idx,
                    cudaStream_t stream);

// Launch counter (the "gpu_launches" the benchmark reports): every kernel launch of this library bumps it.
void count_launch(int n = 1);
int64_t launches_total();

}  // namespace dirb
