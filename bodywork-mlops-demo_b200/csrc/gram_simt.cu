// gram_simt.cu -- CUDA-core Gram accumulator: S += [X 1 y]^T [X 1 y] with fp64 accumulation.
//
// Role: (1) the path for shapes the tensor-core kernel does not take (D % 4 != 0, unaligned
// leading dimension, tiny tranches such as the reference's 1 440-row x 1-feature day,
// stage_3_synthetic_data_generation.py:19); (2) the on-device cross-check of the tensor-core
// kernel.  Products of two fp32 (or bf16) values are exact in fp64, so the only rounding is
// the fp64 running sum -- this matches the numpy float64 oracle to ~1e-15 relative.
//
// Replaces (together with solve.cu): LinearRegression.fit, stage_1_train_model.py:105-106.
#include <cuda_bf16.h>

#include "b2_internal.cuh"

namespace b2 {
namespace {

constexpr int kRB = 32;  // rows per smem tile

template <typename T>
__device__ __forceinline__ float ld_as_float(const T* p);
template <>
__device__ __forceinline__ float ld_as_float<float>(const float* p) { return __ldg(p); }
template <>
__device__ __forceinline__ float ld_as_float<__nv_bfloat16>(const __nv_bfloat16* p) {
  return __bfloat162float(*p);
}

// One thread owns an 8x8 block of S.  nb = ceil((d+2)/8) blocks per side.
template <typename T>
__global__ void __launch_bounds__(320, 1)
gram_simt_kernel(const T* __restrict__ X, const float* __restrict__ y, int64_t n, int d, int64_t ldx,
                 const uint8_t* __restrict__ mask, int keep, double* __restrict__ part) {
  extern __shared__ float tile[];  // [kRB][dp8]
  const int dp = d + 2;
  const int nb = (dp + 7) / 8;
  const int dp8 = nb * 8;
  const int tid = threadIdx.x;
  const bool worker = tid < nb * nb;
  const int bi = worker ? tid / nb : 0;
  const int bj = worker ? tid % nb : 0;

  double acc[8][8];
#pragma unroll
  for (int a = 0; a < 8; ++a)
#pragma unroll
    for (int b = 0; b < 8; ++b) acc[a][b] = 0.0;

  const int64_t n_blocks = (n + kRB - 1) / kRB;
  for (int64_t blk = blockIdx.x; blk < n_blocks; blk += gridDim.x) {
    const int64_t row0 = blk * kRB;
    __syncthreads();
    // cooperative, coalesced tile load; masked / out-of-range rows become all-zero rows
    for (int idx = tid; idx < kRB * dp8; idx += blockDim.x) {
      const int r = idx / dp8, j = idx - r * dp8;
      const int64_t row = row0 + r;
      bool use = row < n;
      if (use && mask != nullptr) use = (mask[row] == (uint8_t)keep);
      float v = 0.f;
      if (use) {
        if (j < d) v = ld_as_float<T>(X + row * ldx + j);
        else if (j == d) v = 1.f;
        else if (j == d + 1) v = __ldg(y + row);
      }
      tile[idx] = v;
    }
    __syncthreads();
    if (worker) {
#pragma unroll 4
      for (int r = 0; r < kRB; ++r) {
        const float4* ra = reinterpret_cast<const float4*>(tile + r * dp8 + bi * 8);
        const float4* rb = reinterpret_cast<const float4*>(tile + r * dp8 + bj * 8);
        const float4 a0 = ra[0], a1 = ra[1], b0 = rb[0], b1 = rb[1];
        const double av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
        const double bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
        for (int a = 0; a < 8; ++a)
#pragma unroll
          for (int b = 0; b < 8; ++b) acc[a][b] = fma(av[a], bv[b], acc[a][b]);
      }
    }
  }
  if (worker) {
    double* out = part + (size_t)blockIdx.x * kMaxS * kMaxS;
#pragma unroll
    for (int a = 0; a < 8; ++a) {
      const int ia = bi * 8 + a;
#pragma unroll
      for (int b = 0; b < 8; ++b) {
        const int jb = bj * 8 + b;
        if (ia < dp && jb < dp) out[ia * dp + jb] = acc[a][b];
      }
    }
  }
}

// S[a][b] (+)= sum over CTAs (fixed order -> deterministic); assign: S = sum (a fresh statistic)
__global__ void gram_simt_reduce(const double* __restrict__ part, int n_ctas, int dp, int assign,
                                 double* __restrict__ S) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= dp * dp) return;
  double s = 0.0;
  for (int c = 0; c < n_ctas; ++c) s += part[(size_t)c * kMaxS * kMaxS + idx];
  S[idx] = assign ? s : S[idx] + s;
}

}  // namespace

int launch_gram_simt(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n, int d,
                     int64_t ldx, const uint8_t* mask, int keep, bool assign) {
  if (n <= 0) return B2_OK;
  const int dp = d + 2;
  const int nb = (dp + 7) / 8;
  const int dp8 = nb * 8;
  const int threads = ((nb * nb + 31) / 32) * 32;
  const int64_t n_blocks = (n + kRB - 1) / kRB;
  const int grid = (int)(n_blocks < ctx->simt_ctas ? n_blocks : ctx->simt_ctas);
  const size_t smem = sizeof(float) * kRB * dp8;
  if (x_dtype == B2_F32) {
    gram_simt_kernel<float><<<grid, threads, smem, ctx->stream>>>(
        static_cast<const float*>(X), y, n, d, ldx, mask, keep, ctx->simt_part);
  } else {
    gram_simt_kernel<__nv_bfloat16><<<grid, threads, smem, ctx->stream>>>(
        static_cast<const __nv_bfloat16*>(X), y, n, d, ldx, mask, keep, ctx->simt_part);
  }
  B2_CUDA(cudaGetLastError());
  gram_simt_reduce<<<(dp * dp + 255) / 256, 256, 0, ctx->stream>>>(ctx->simt_part, grid, dp, assign ? 1 : 0, ctx->S);
  B2_CUDA(cudaGetLastError());
  ctx->launches += 2;
  return B2_OK;
}

}  // namespace b2
