// b2_dmma.cuh -- the fp64 tensor-core MMA and the per-element row load of the fp64 row passes (ridge_loo.cu,
// score_std.cu, glm.cu).
#pragma once
#include <cuda_bf16.h>

namespace b2 {

__device__ __forceinline__ void dmma(double& c0, double& c1, double a, double b) {
  // fragments (PTX mma.m8n8k4.f64): A row = lane / 4, col = lane % 4; B row(k) = lane % 4, col(n) = lane / 4;
  // C row = lane / 4, cols = 2 (lane % 4) + {0, 1}
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
               : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}

template <typename T>
__device__ __forceinline__ float ld_row_val(const T* __restrict__ p);
template <>
__device__ __forceinline__ float ld_row_val<float>(const float* __restrict__ p) { return __ldg(p); }
template <>
__device__ __forceinline__ float ld_row_val<__nv_bfloat16>(const __nv_bfloat16* __restrict__ p) {
  return __bfloat162float(*p);
}

}  // namespace b2
