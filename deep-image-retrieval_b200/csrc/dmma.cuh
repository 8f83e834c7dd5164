// cp.async staging and the fp64 tensor-core MMA (mma.sync m16n8k16 .f64, native DMMA on sm_90), shared by the fp64
// GEMMs of label_count.cu (threshold counts) and pca.cu (covariance Gram).
#pragma once
#include <stdint.h>

namespace dirb {

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, bool pred) {
  const uint32_t s = static_cast<uint32_t>(__cvta_generic_to_shared(smem));
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(s), "l"(gmem), "r"(pred ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// D (16x8, fp64) += A (16x16, row) * B (16x8, col).  Fragments (g = lane / 4, t = lane % 4):
//   a[i] = A[g + 8 (i % 2)][t + 4 (i / 2)],  b[i] = B[t + 4 i][g],  c[i] = C[g + 8 (i / 2)][2 t + i % 2].
__device__ __forceinline__ void dmma16816(double (&c)[4], const double (&a)[8], const double (&b)[4]) {
  asm("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, "
      "{%12,%13,%14,%15}, {%0,%1,%2,%3};"
      : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
      : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]), "d"(b[1]),
        "d"(b[2]), "d"(b[3]));
}

}  // namespace dirb
