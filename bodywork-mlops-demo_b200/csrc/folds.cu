// folds.cu -- the two small kernels of b2_gram_folds (DESIGN.md section 8).
//
//   fold_range_kernel : first and last row of every fold, from fold ids in device memory.  Each thread walks a run of
//                       kRangeRows consecutive ids and records only where a fold's stretch starts and ends, into the
//                       CTA's shared copy; the CTA then merges the folds it saw into the global ranges.  Contiguous folds
//                       cost one shared atomic per thread, shuffled ones one per change of id.
//   fold_sum_kernel   : S = sum of the fold statistics, added in fold order from 0 -- the additions solve_enet_kernel
//                       makes when it sums the folds itself, so the refit's S and the grid of every path agree bit for bit.
#include "b2_internal.cuh"

namespace b2 {
namespace {

constexpr int kRangeThreads = 256;
constexpr int kRangeRows = 64;

// range[2 k] = max over rows of fold k of (n - row), range[2 k + 1] = max of (row + 1): no initial value other than 0
__global__ void __launch_bounds__(kRangeThreads)
fold_range_kernel(const uint8_t* __restrict__ ids, int64_t n, int n_folds, unsigned long long* __restrict__ range) {
  __shared__ unsigned long long loc[2 * kMaxFolds];
  for (int i = threadIdx.x; i < 2 * n_folds; i += blockDim.x) loc[i] = 0ull;
  __syncthreads();
  const int64_t r0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * kRangeRows;
  const int64_t r1 = r0 + kRangeRows < n ? r0 + kRangeRows : n;
  if (r0 < n) {
    int cur = ids[r0];
    int64_t start = r0;
    for (int64_t r = r0 + 1; r <= r1; ++r) {
      const int f = r < r1 ? ids[r] : -1;
      if (f != cur) {
        if (cur < n_folds) {
          atomicMax(&loc[2 * cur], (unsigned long long)(n - start));
          atomicMax(&loc[2 * cur + 1], (unsigned long long)r);
        }
        cur = f;
        start = r;
      }
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 2 * n_folds; i += blockDim.x)
    if (loc[i] != 0ull) atomicMax(&range[i], loc[i]);
}

__global__ void fold_sum_kernel(const double* __restrict__ folds, int n_folds, int count, double* __restrict__ S) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  double t = 0.0;
  for (int j = 0; j < n_folds; ++j) t += folds[(size_t)j * count + i];
  S[i] = t;
}

}  // namespace

int launch_fold_ranges(b2_ctx* ctx, const uint8_t* fold_of_row, int64_t n, int n_folds, unsigned long long* range) {
  B2_CUDA(cudaMemsetAsync(range, 0, sizeof(unsigned long long) * 2 * n_folds, ctx->stream));
  const int64_t per_cta = (int64_t)kRangeThreads * kRangeRows;
  const int64_t ctas = (n + per_cta - 1) / per_cta;
  if (ctas > 0) {
    fold_range_kernel<<<(unsigned int)ctas, kRangeThreads, 0, ctx->stream>>>(fold_of_row, n, n_folds, range);
    B2_CUDA(cudaGetLastError());
    ctx->launches += 1;
  }
  return B2_OK;
}

int launch_fold_sum(b2_ctx* ctx, const double* folds, int n_folds, int d, double* S) {
  const int count = (d + 2) * (d + 2);
  fold_sum_kernel<<<(count + 255) / 256, 256, 0, ctx->stream>>>(folds, n_folds, count, S);
  B2_CUDA(cudaGetLastError());
  ctx->launches += 1;
  return B2_OK;
}

}  // namespace b2
