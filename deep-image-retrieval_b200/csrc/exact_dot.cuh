// The library's exact score of one (query, row) pair.
#pragma once

namespace dirb {

// Exact score of one (query, row) pair by one warp: fp64 accumulation of the fp32 products, fixed summation order
// (lane-strided float4 loads, xor-shuffle tree).  The exact scores of the search, the rank counts and the label counts
// all come from this function, so two evaluations of the same pair - or of two identical rows - are bit-identical
// wherever they are computed.  (scores_exact_kernel, the dense matrix behind common.matmul, sums each float4's four
// products before adding them to its accumulator: its fp32 outputs can differ from fl32(exact_dot_warp) in the last
// bit, for roughly 1e-7 of the pairs.)
__device__ __forceinline__ double exact_dot_warp(const float* __restrict__ qrow, const float* __restrict__ dbrow, int D,
                                                 int lane) {
  const float4* a = reinterpret_cast<const float4*>(qrow);
  const float4* b = reinterpret_cast<const float4*>(dbrow);
  double acc = 0.0;
  for (int i = lane; i < D / 4; i += 32) {
    const float4 x = __ldg(a + i), y = __ldg(b + i);
    acc += static_cast<double>(x.x) * y.x;
    acc += static_cast<double>(x.y) * y.y;
    acc += static_cast<double>(x.z) * y.z;
    acc += static_cast<double>(x.w) * y.w;
  }
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  return acc;
}

}  // namespace dirb
