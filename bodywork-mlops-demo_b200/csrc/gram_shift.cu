// gram_shift.cu -- the per-column shift c of the approximate Gram paths (tensor core and narrow rows).
//
// Both paths accumulate moments of the shifted rows v = x - c, y' = y - c_y in fp32 and undo the shift in fp64
// (b2_shift.cuh).  Any c is algebraically exact; a c near the column mean keeps |v| / sigma small, which is what the
// fp32 products and the bf16 operand split need.  c is the mean of the finite block means of a strided sample of at
// most 2048 rows, split over 64 blocks.  It stays fp32 for fp32 rows: the operands carry |x - c| / sigma, so a c
// rounded to bf16 (spacing 64 at a column mean of 1e4) would cost digits wherever a column's mean is large against its
// spread.  For bf16 rows the feature shifts are rounded to bf16, so that x and c share one grid and x - c is exact.
//
// ctx->shift: c[kMaxD + 1] (features, zero from d on, c_y at kMaxD), then the 64 partial means, then the ticket counter.
#include <cuda_bf16.h>

#include "b2_internal.cuh"
#include "b2_ptx.cuh"

namespace b2 {
namespace {

constexpr int kShiftBlocks = 64;                 // partial means of the row sample, one per block
constexpr int kShiftStride = kMaxD + 1;          // floats per partial: features, then y (slot kMaxD)
constexpr int kShiftPartOff = kMaxD + 1;         // partials follow c
constexpr int kShiftTicketOff = kShiftPartOff + kShiftBlocks * kShiftStride;

__host__ __device__ __forceinline__ int64_t shift_samples(int64_t n) { return n < 2048 ? n : 2048; }

__device__ __forceinline__ float shift_round(float c, bool round_bf16) {
  return round_bf16 ? __bfloat162float(__float2bfloat16_rn(c)) : c;
}
// c_j from the 64 partial means (NaN: a block without a finite sample).  noinline: inlined into the last block's tail,
// it makes ptxas give the kernel 32 instead of 71 registers and spread the sample loop's 8 loads between dependent adds.
__device__ __noinline__ float shift_value(const float* sp, int j, bool round_bf16) {
  float acc = 0.f;
  int cnt = 0;
#pragma unroll 8
  for (int b = 0; b < kShiftBlocks; ++b) {
    const float p = sp[b * kShiftStride + j];
    if (p == p) { acc += p; ++cnt; }
  }
  return shift_round(cnt > 0 ? acc / (float)cnt : 0.f, round_bf16);
}

// 64 blocks x (4 row groups x 160 columns): a thread sums 8 sample rows (one batch of loads in flight -- the rows are
// megabytes apart, every load is a DRAM round trip), the 4 groups are combined in a fixed order.  The last block to
// finish (ticket) combines the 64 partial means into c and re-arms the ticket.
constexpr int kShiftCols = 160;                  // >= kMaxD + 1, a multiple of 32
constexpr int kShiftGroups = 4;

template <typename T>
__global__ void __launch_bounds__(kShiftCols * kShiftGroups)
tc_shift_kernel(const T* __restrict__ X, const float* __restrict__ y, int64_t n, int d, int64_t ldx, float* shift) {
  __shared__ float sub[kShiftGroups][kShiftCols];
  __shared__ int subn[kShiftGroups][kShiftCols];
  __shared__ bool last_block;
  __shared__ float part_s[kShiftBlocks * kShiftStride];   // the last block's copy of the partials (33 KB)
  float* sp = shift + kShiftPartOff;
  const int j = threadIdx.x % kShiftCols, g = threadIdx.x / kShiftCols;
  const int64_t samples = shift_samples(n);
  const int64_t stride = n / samples;
  const int64_t per = (samples + kShiftBlocks - 1) / kShiftBlocks;
  const int64_t s0 = blockIdx.x * per;
  const int64_t s1 = (s0 + per < samples) ? s0 + per : samples;
  float acc = 0.f;
  int cnt = 0;
  if (j <= d) {
#pragma unroll 8
    for (int64_t s = s0 + g; s < s1; s += kShiftGroups) {
      const int64_t row = s * stride;
      const float v = (j < d) ? raw_ld_global<T>(X + row * ldx + j) : __ldg(y + row);
      const bool finite = fabsf(v) <= 3.0e38f;    // the sample ignores the row mask: a dropped row may hold NaN / Inf
      acc += finite ? v : 0.f;
      cnt += finite ? 1 : 0;
    }
  }
  sub[g][j] = acc;
  subn[g][j] = cnt;
  __syncthreads();
  if (g == 0 && j <= d) {
    const int c = subn[0][j] + subn[1][j] + subn[2][j] + subn[3][j];
    sp[blockIdx.x * kShiftStride + (j == d ? kMaxD : j)] =
        c > 0 ? (((sub[0][j] + sub[1][j]) + sub[2][j]) + sub[3][j]) / (float)c : __int_as_float(0x7fc00000);
    __threadfence();
  }
  __syncthreads();
  unsigned int* ticket = reinterpret_cast<unsigned int*>(shift + kShiftTicketOff);
  if (threadIdx.x == 0) last_block = atomicAdd(ticket, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!last_block) return;
  __threadfence();
  // the partials of the d + 1 sampled columns into shared memory, 16 loads in flight per thread: read where they are
  // summed, they would cost one L2 round trip per batch of 8
  if (j <= d) {
    const int col = j == d ? kMaxD : j;
    float p[kShiftBlocks / kShiftGroups];
#pragma unroll
    for (int i = 0; i < kShiftBlocks / kShiftGroups; ++i) p[i] = __ldcg(sp + (g + kShiftGroups * i) * kShiftStride + col);
#pragma unroll
    for (int i = 0; i < kShiftBlocks / kShiftGroups; ++i) part_s[(g + kShiftGroups * i) * kShiftStride + col] = p[i];
  }
  __syncthreads();
  for (int k = threadIdx.x; k <= kMaxD; k += blockDim.x)
    shift[k] = k == kMaxD ? shift_value(part_s, kMaxD, false) : (k < d ? shift_value(part_s, k, sizeof(T) == 2) : 0.f);
  if (threadIdx.x == 0) *ticket = 0u;
}

}  // namespace

size_t gram_shift_bytes() { return sizeof(float) * (kShiftTicketOff + 1); }

int launch_gram_shift(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n, int d, int64_t ldx) {
  if (x_dtype == B2_F32)
    tc_shift_kernel<float><<<kShiftBlocks, kShiftCols * kShiftGroups, 0, ctx->stream>>>(
        static_cast<const float*>(X), y, n, d, ldx, ctx->shift);
  else
    tc_shift_kernel<__nv_bfloat16><<<kShiftBlocks, kShiftCols * kShiftGroups, 0, ctx->stream>>>(
        static_cast<const __nv_bfloat16*>(X), y, n, d, ldx, ctx->shift);
  B2_CUDA(cudaGetLastError());
  ctx->launches += 1;
  return B2_OK;
}

}  // namespace b2
