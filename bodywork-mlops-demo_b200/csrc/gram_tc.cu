// gram_tc.cu -- the hot kernel: row-block streaming Gram accumulator on the Hopper tensor core (wgmma, sm_90a).
//
// Replaces the pass over the training rows inside LinearRegression.fit
// (stage_1_train_model.py:105-106 -> sklearn/linear_model/_base.py: centre + LAPACK gelsd).
//
// Data flow per CTA (persistent, one CTA per SM, contiguous range of 64-row tiles):
//
//   HBM --TMA (cp.async.bulk.tensor, evict-first)--> smem raw tile [64 rows][D] (+ y, + row mask)
//     --6 transform warps: v = x - c (per-column shift), bf16 split v = hi + lo
//     -- 1 "E" warp: extra columns E = [1, y'_hi, y'_lo] (y' = y - c_y), CUDA-core sums of y', y'^2, rows
//     --> operands, K-major canonical layout (8 x 16 B core matrices, no swizzle; one 16-byte chunk =
//         8 consecutive rows of X for one feature), per 8-row K group:
//            rows j = 0..127 hi | 128..143 E | 144..271 lo          (B = [hi | E], A = hi or A = lo)
//     --wgmma.mma_async m64n144k16 (bf16 x bf16 -> fp32 in registers); warpgroup c (c = 0, 1) owns features
//       64c..64c+63 of both accumulators, two wgmma per K step of 16 rows:
//            D1[i][j] += sum_r hi[r][i] * [hi | E][r][j]      drained every `drain_rows` rows
//            D2[i][j] += sum_r lo[r][i] * [hi | E][r][j]      small zero-mean terms: drained once at the end
//        so D1[:, :128] = hi^T hi, D2[:, :128] = lo^T hi, column 128 = sum v, columns 129/130 = sum v*y'.
//     --every `drain_rows` rows the two consumer warpgroups fold D1 into this CTA's fp64 partial in global
//        memory (L2-resident) and restart it from zero; the producer warps keep filling stages meanwhile.
//       The 144 accumulator registers per consumer thread come from the producers (setmaxnreg).
//
// Why the shift and the split: the tensor core accumulates fp32 with truncation, so raw (uncentred)
// second moments cannot reach the 1e-4 coefficient tolerance; after the shift the Gram is ~diagonal and
// the centring in the solve subtracts almost nothing.  hi+lo carries 16 mantissa bits, i.e. products are
// accurate to ~2^-17 relative (lo*lo is dropped).
//
// tc_reduce_kernel sums the per-CTA partials in a fixed order (deterministic); tc_fold_kernel undoes the shift
// in fp64 and adds the result to the context's raw statistic S = [X 1 y]^T [X 1 y].
#include <cuda_bf16.h>
#include <stdlib.h>

#include "b2_internal.cuh"
#include "b2_ptx.cuh"
#include "b2_xchg.cuh"

namespace b2 {
namespace {

// ------------------------------------------------------------------------------------------
// geometry
// ------------------------------------------------------------------------------------------
constexpr int kRawStages = 4;
constexpr int kOpStages = 2;
constexpr int kConsumerWGs = 2;                    // warpgroups 0-1: wgmma + drain, 64 features each
constexpr int kXformWarps = 6;
constexpr int kThreads = 128 * (kConsumerWGs + 2); // warps: 0-7 consumers, 8 TMA, 9 E, 10-15 transform
constexpr int kTmaWarp = 4 * kConsumerWGs, kEWarp = kTmaWarp + 1, kFirstXformWarp = kTmaWarp + 2;
static_assert(kFirstXformWarp + kXformWarps == kThreads / 32, "warp roles");
constexpr int kProducers = kXformWarps + 1;        // arrivals that fill an operand stage (transform warps + E warp)
constexpr int kConsumerWarps = 4 * kConsumerWGs;   // arrivals that free an operand stage
constexpr uint32_t kConsumerRegs = 200, kProducerRegs = 56;   // setmaxnreg split of the 128 x 512 register file
static_assert(kConsumerRegs * 128 * kConsumerWGs + kProducerRegs * (kThreads - 128 * kConsumerWGs) <= 65536,
              "register budget");
constexpr int kAccRegs = kTcN / 2;                 // fp32 accumulator registers per thread (64 x 144 per warpgroup)
constexpr int kKGroups = kTcRows / 8;              // 8-row K groups per stage
constexpr uint32_t kRawStageBytes = kTcRows * kMaxD * 4;      // 32768 (fp32, D = 128)
constexpr uint32_t kOpSBO = 128;                              // bytes between 8-row j groups (core matrices along M/N)
constexpr uint32_t kOpLBO = (16 + 2 + 16) * kOpSBO;           // 4352: hi | E | lo groups per K group
constexpr uint32_t kOpEOff = 16 * kOpSBO;                     // E block inside a K group
constexpr uint32_t kOpLoOff = 18 * kOpSBO;                    // lo block inside a K group
constexpr uint32_t kOpStageBytes = kKGroups * kOpLBO;         // 34816
constexpr uint32_t kOffRaw = 0;
constexpr uint32_t kOffOp = kOffRaw + kRawStages * kRawStageBytes;     // 131072
constexpr uint32_t kOffY = kOffOp + kOpStages * kOpStageBytes;         // 200704
constexpr int kMaxPack = 5;                                             // original rows per 128-wide super-row (3 E columns each)
constexpr uint32_t kYStageBytes = kTcRows * kMaxPack * 4;               // 1280
constexpr uint32_t kMStageBytes = 384;                                  // 64 * kMaxPack = 320 mask bytes, padded: TMA
                                                                        // destinations are 128-byte aligned
static_assert(kMStageBytes >= kTcRows * kMaxPack && kMStageBytes % 128 == 0 && kYStageBytes % 128 == 0, "stage alignment");
constexpr uint32_t kOffMask = kOffY + kRawStages * kYStageBytes;
constexpr uint32_t kOffBar = kOffMask + kRawStages * kMStageBytes;
constexpr int kNumBars = 2 * kRawStages + 2 * kOpStages;
constexpr uint32_t kOffShift = kOffBar + kNumBars * 8;
constexpr uint32_t kSmemBytes = kOffShift + (kMaxD + 4) * 4 + 1024;    // + alignment slack (~204 KB)
static_assert(kSmemBytes <= 227 * 1024, "shared memory budget");

// ------------------------------------------------------------------------------------------
// PTX wrappers
// ------------------------------------------------------------------------------------------
constexpr uint64_t kEvictFirst = 0x12F0000000000000ull;  // L2 cache hint: streaming data, read once

__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* tm, int c0, int c1, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4}], [%2], %5;" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(tm)), "r"(bar), "r"(c0), "r"(c1), "l"(kEvictFirst)
      : "memory");
}
__device__ __forceinline__ void tma_load_1d(uint32_t dst, const CUtensorMap* tm, int c0, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.1d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3}], [%2], %4;" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(tm)), "r"(bar), "r"(c0), "l"(kEvictFirst)
      : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* tm) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tm)) : "memory");
}

// K-major, no-swizzle ("interleave") wgmma shared-memory matrix descriptor: start address, LBO = bytes between the two
// core matrices along K (one K group to the next), SBO = bytes between 8-row core matrices along M / N
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t addr) {
  return (uint64_t)((addr & 0x3FFFFu) >> 4) | ((uint64_t)(kOpLBO >> 4) << 16) | ((uint64_t)(kOpSBO >> 4) << 32);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across a wgmma fence or wait
template <int N>
__device__ __forceinline__ void fence_regs(float (&r)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(r[i])::"memory");
}
// D[64 x 144] (+)= A[64 x 16] * B[16 x 144]: bf16 operands from shared memory (both K-major), fp32 accumulators in
// registers (wgmma fragment layout); scale_d = 0 overwrites D.  Issued by all 128 threads of a warpgroup.
__device__ __forceinline__ void wgmma_m64n144k16(float (&d)[72], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %74, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n144k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, "
      " %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
      " %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, "
      " %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      " %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, "
      " %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71}, "
      "%72, %73, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71])
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
}
// D[64 x 128] (+)= A[64 x 16] * B[16 x 128]: A K-major, B MN-major (the raw 128B-swizzled TMA tile)
__device__ __forceinline__ void wgmma_m64n128k16_bmn(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      " %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      " %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      " %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, 0, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
}
// D[64 x 16] (+)= A[64 x 16] * B[16 x 16]: both K-major (B = the E columns)
__device__ __forceinline__ void wgmma_m64n16k16(float (&d)[8], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7}, "
      "%8, %9, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
}
// MN-major, 128B-swizzled descriptor of the raw bf16 tile of the D = 128 bf16 path: two TMA boxes of [64 rows][64
// features] (128-byte rows, 8-row swizzle atoms of 1024 bytes); LBO = bytes from features 0..63 to 64..127 (one box),
// SBO = bytes from one 8-row K group to the next
constexpr uint32_t kRawBoxBytes = kTcRows * 64 * 2;   // 8192
__device__ __forceinline__ uint64_t make_raw_desc(uint32_t addr) {
  return (uint64_t)((addr & 0x3FFFFu) >> 4) | ((uint64_t)(kRawBoxBytes >> 4) << 16) | ((uint64_t)(1024u >> 4) << 32) |
         (1ull << 62);
}

__device__ __forceinline__ void st_shared_v4(uint32_t addr, const uint32_t (&v)[4]) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v[0]), "r"(v[1]), "r"(v[2]), "r"(v[3])
               : "memory");
}
__device__ __forceinline__ void st_shared_u16(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.u16 [%0], %1;" ::"r"(addr), "h"((unsigned short)v) : "memory");
}
// bf16 split of two fp32 values: hi = rn(v), lo = rn(v - hi), packed (element 0 in the low half)
__device__ __forceinline__ void split2(float v0, float v1, uint32_t& hi, uint32_t& lo) {
  const __nv_bfloat162 h = __floats2bfloat162_rn(v0, v1);
  hi = *reinterpret_cast<const uint32_t*>(&h);
  const float h0 = __uint_as_float(hi << 16), h1 = __uint_as_float(hi & 0xffff0000u);
  const __nv_bfloat162 l = __floats2bfloat162_rn(v0 - h0, v1 - h1);
  lo = *reinterpret_cast<const uint32_t*>(&l);
}

// ------------------------------------------------------------------------------------------
// per-column shift c: mean of a strided row sample (any value near the column mean will do;
// the algebra in tc_fold_kernel is exact for every c)
// ------------------------------------------------------------------------------------------
constexpr int kShiftBlocks = 64;                 // partial sums of the row sample, one per block
constexpr int kShiftStride = kMaxD + 1;          // floats per partial: features, then y (slot kMaxD)

__host__ __device__ __forceinline__ int64_t shift_samples(int64_t n) { return n < 2048 ? n : 2048; }

// c_j from the 64 partial sums; bf16-representable so that (bf16 input - c) is exact in fp32.
// Called with identical arguments by the Gram kernel and by tc_fold_kernel -> identical c.
__device__ __forceinline__ float shift_value(const float* __restrict__ sp, int j, int64_t n) {
  float acc = 0.f;
#pragma unroll 8
  for (int b = 0; b < kShiftBlocks; ++b) acc += sp[b * kShiftStride + j];
  return __bfloat162float(__float2bfloat16_rn(acc / (float)shift_samples(n)));
}

// 64 blocks x (4 row groups x 160 columns): a thread sums 8 sample rows (one batch of loads in flight -- the rows are
// megabytes apart, every load is a DRAM round trip), the 4 groups are combined in a fixed order.
constexpr int kShiftCols = 160;                  // >= kMaxD + 1, a multiple of 32
constexpr int kShiftGroups = 4;

template <typename T>
__global__ void __launch_bounds__(kShiftCols * kShiftGroups)
tc_shift_kernel(const T* __restrict__ X, const float* __restrict__ y, int64_t n, int d,
                int64_t ldx, float* __restrict__ sp) {
  __shared__ float sub[kShiftGroups][kShiftCols];
  const int j = threadIdx.x % kShiftCols, g = threadIdx.x / kShiftCols;
  const int64_t samples = shift_samples(n);
  const int64_t stride = n / samples;
  const int64_t per = (samples + kShiftBlocks - 1) / kShiftBlocks;
  const int64_t s0 = blockIdx.x * per;
  const int64_t s1 = (s0 + per < samples) ? s0 + per : samples;
  float acc = 0.f;
  if (j <= d) {
#pragma unroll 8
    for (int64_t s = s0 + g; s < s1; s += kShiftGroups) {
      const int64_t row = s * stride;
      const float v = (j < d) ? raw_ld_global<T>(X + row * ldx + j) : __ldg(y + row);
      acc += (fabsf(v) <= 3.0e38f) ? v : 0.f;     // the sample ignores the row mask: a dropped row may hold NaN / Inf
    }
  }
  sub[g][j] = acc;
  __syncthreads();
  if (g == 0 && j <= d) sp[blockIdx.x * kShiftStride + (j == d ? kMaxD : j)] = ((sub[0][j] + sub[1][j]) + sub[2][j]) + sub[3][j];
}

// ------------------------------------------------------------------------------------------
// finalize, shared by the stand-alone kernels (tc_reduce_kernel / tc_fold_kernel: the b2_gram_accumulate path) and
// by the fused tail of the Gram kernel (b2_fit): the same summation order in both, so the two paths agree bit for bit.
//   red[col * 128 + i], col in [0, 288):  col < 144: D1 (A = hi), col >= 144: D2 (A = lo), columns of [hi | E]
//   red[kTcAccElems + 0..2]            : sum y', sum y'^2, rows used
// ------------------------------------------------------------------------------------------
constexpr int kRedElems = kTcAccElems + 3;

// Sum over the CTAs of elements [e0, e1) of the per-CTA partials.  4 threads per element: thread (e, q) sums the q-th
// quarter of the CTAs with 8 loads in flight (the loads are the latency), the quarters are combined in the fixed order
// 0..3 -> deterministic.  `quarter`: shared scratch of 4 * (blockDim.x / 4) doubles.  Call with the whole block.
__device__ __forceinline__ void tc_reduce_range(const double* part, const double* side, int n_ctas, double* red,
                                                int e0, int e1, double* quarter) {
  const int epb = blockDim.x >> 2;                 // elements per pass
  const int e = threadIdx.x % epb, q = threadIdx.x / epb;
  const int per = (n_ctas + 3) / 4;
  const int c0 = q * per, c1 = (c0 + per < n_ctas) ? c0 + per : n_ctas;
  for (int base = e0; base < e1; base += epb) {
    const int idx = base + e;
    if (idx < e1 && idx < kTcAccElems) {
      double acc[8] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
      int c = c0;
      for (; c + 8 <= c1; c += 8) {
#pragma unroll
        for (int u = 0; u < 8; ++u) acc[u] += __ldcg(part + (size_t)(c + u) * kTcAccElems + idx);
      }
      for (; c < c1; ++c) acc[0] += __ldcg(part + (size_t)c * kTcAccElems + idx);
      quarter[q * epb + e] = ((acc[0] + acc[1]) + (acc[2] + acc[3])) + ((acc[4] + acc[5]) + (acc[6] + acc[7]));
    } else if (idx < e1 && idx < kRedElems) {
      // the three CUDA-core sums (sum y', sum y'^2, rows): same quarter scheme, loads 8 deep (a serial walk over the
      // CTAs costs one L2 round trip each, ~140 ns per CTA)
      const int k = idx - kTcAccElems;
      double acc[8] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
      int c = c0;
      for (; c + 8 <= c1; c += 8) {
#pragma unroll
        for (int u = 0; u < 8; ++u)
          acc[u] += __ldcg(side + (size_t)(c + u) * kTcSideDoubles + k) + __ldcg(side + (size_t)(c + u) * kTcSideDoubles + 3 + k);
      }
      for (; c < c1; ++c) acc[0] += __ldcg(side + (size_t)c * kTcSideDoubles + k) + __ldcg(side + (size_t)c * kTcSideDoubles + 3 + k);
      quarter[q * epb + e] = ((acc[0] + acc[1]) + (acc[2] + acc[3])) + ((acc[4] + acc[5]) + (acc[6] + acc[7]));
    }
    __syncthreads();
    if (q == 0 && idx < e1 && idx < kRedElems)
      red[idx] = ((quarter[e] + quarter[epb + e]) + quarter[2 * epb + e]) + quarter[3 * epb + e];
    __syncthreads();
  }
}

// Grid-wide barrier of a co-resident (cooperatively launched) grid: arrive on a counter, wait until all CTAs have.
// The counter is zeroed again by the kernel's final ticket.  Bounded: a protocol bug traps instead of hanging.
__device__ __forceinline__ void grid_barrier(unsigned int* ctr) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(ctr, 1u);
    const uint64_t t0 = globaltimer_ns();
    unsigned int seen;
    do {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(seen) : "l"(ctr) : "memory");
      if (seen < gridDim.x) {
        __nanosleep(40);
        if (globaltimer_ns() - t0 > 4000000000ull) __trap();
      }
    } while (seen < gridDim.x);
    __threadfence();
  }
  __syncthreads();
}

// `pack` original rows share one 128-wide super-row (d * pack == 128 when pack > 1): original feature a of
// sub-row blk is super-feature blk*d + a, and its E columns are 128 + 3*blk (+0 ones, +1 y'_hi, +2 y'_lo).
// The true statistic is the sum over blk of the diagonal (blk, blk) blocks.
// Returns the contribution of this launch to S[idx]; c[j] = the shift of feature j, c[kMaxD] = the shift of y
// (fp64 copy in `red` for the stand-alone kernel, the CTA's fp32 smem copy in the fused tail -- the same values).
template <typename CT>
__device__ __forceinline__ double tc_fold_value(const double* red, const CT* c, int d, int pack, int idx) {
  const int dp = d + 2;
  const int a = idx / dp, b = idx % dp;
  // D1[i][j] = red[j*128 + i], D2[i][j] = red[(144 + j)*128 + i]
  auto D1 = [&](int i, int j) { return __ldcg(red + (size_t)j * kTcM + i); };
  auto D2 = [&](int i, int j) { return __ldcg(red + (size_t)(kTcN + j) * kTcM + i); };
  auto s1 = [&](int i) {                                                     // sum (x_i - c_i)
    double t = 0.0;
    for (int blk = 0; blk < pack; ++blk) t += D1(blk * d + i, 128 + 3 * blk) + D2(blk * d + i, 128 + 3 * blk);
    return t;
  };
  auto sxy = [&](int i) {                                                    // sum (x_i - c_i) y'
    double t = 0.0;
    for (int blk = 0; blk < pack; ++blk) {
      const int r = blk * d + i, e = 128 + 3 * blk;
      t += D1(r, e + 1) + D1(r, e + 2) + D2(r, e + 1) + D2(r, e + 2);
    }
    return t;
  };
  const double sy = __ldcg(red + kTcAccElems + 0);
  const double syy = __ldcg(red + kTcAccElems + 1);
  const double n = __ldcg(red + kTcAccElems + 2);
  const double cy = (double)c[kMaxD];
  double val;
  if (a < d && b < d) {
    const double ca = (double)c[a], cb = (double)c[b];
    // G'(a,b) = sum (x_a-c_a)(x_b-c_b) ~= hi.hi + lo.hi + hi.lo   (lo.lo dropped, ~2^-18 relative)
    double g = 0.0;
    for (int blk = 0; blk < pack; ++blk) {
      const int ia = blk * d + a, ib = blk * d + b;
      g += 0.5 * (D1(ia, ib) + D1(ib, ia)) + D2(ia, ib) + D2(ib, ia);
    }
    val = g + ca * s1(b) + cb * s1(a) + n * ca * cb;
  } else if (a < d || b < d) {
    const int i = a < d ? a : b;
    const int o = a < d ? b : a;  // d (ones) or d+1 (y)
    const double ci = (double)c[i];
    if (o == d) val = s1(i) + n * ci;
    else val = sxy(i) + cy * s1(i) + ci * sy + n * ci * cy;
  } else if (a == d && b == d) {
    val = n;
  } else if (a == d + 1 && b == d + 1) {
    val = syy + 2.0 * cy * sy + n * cy * cy;
  } else {
    val = sy + n * cy;
  }
  return val;
}

// ------------------------------------------------------------------------------------------
// the Gram kernel
// ------------------------------------------------------------------------------------------
// DFIX = 128: feature count known at compile time (immediate smem offsets, no index arithmetic in
// the transform loop); DFIX = 0: runtime d (any multiple of 4 / 8 up to 128).
// SPLIT = true : operands hi + lo (16 mantissa bits, the default);
// SPLIT = false: single bf16 operand hi = rn(x - c) ("bf16-accum" mode of BASELINE.json configs[1]): half the MMAs,
//                no lo arithmetic; the operand rounding error (2^-9 relative, zero mean) averages out as 1/sqrt(n).
// RAWB (bf16 rows, D = 128, no packing): the raw TMA tile itself (128B-swizzled) is the B operand, so the transform
//   writes only the A operands.  D1[i][j] = sum_r hi[r][i] x[r][j] (raw, unshifted x) and E1[i][e] = sum_r hi[r][i] E[r][e];
//   the drain subtracts c_j * sum_r hi[r][i] (the ones column of E1), which leaves sum hi_i v_j with the B side exact.
//   lo has its own accumulators (D2, E2, small zero-mean sums, drained once at the end), stored halved in the feature
//   columns so that the fold's D2(a,b) + D2(b,a) adds sum lo_a v_b once, symmetrised -- the partial means what the other
//   variants' partials mean.  The raw stage is
//   held until the MMAs have read it; masked-out rows are zeroed in it (0 * NaN would poison the sums).
template <typename T, int DFIX, bool SPLIT, bool RAWB = false>
__global__ void __launch_bounds__(kThreads, 1)
gram_tc_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmY,
               const __grid_constant__ CUtensorMap tmM, int y_map_2d, int has_mask, int keep,
               int64_t n_rows, int d_arg, int pack, int d_orig, int64_t n_shift, const float* __restrict__ shift,
               int chunk_tiles,
               double* __restrict__ part, double* __restrict__ side, uint32_t wait_ns, uint32_t dbg_arg) {
#ifdef B2_DEV_KNOBS
  const uint32_t dbg = dbg_arg;      // ablation switches (tools/build_dev.sh): results are WRONG when non-zero
#else
  constexpr uint32_t dbg = 0u;       // product build: the ablation branches compile away
  (void)dbg_arg;
#endif
  const int d = DFIX ? DFIX : d_arg;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem = smem_raw + (sbase - smem_u32(smem_raw));
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  const uint32_t bar_raw_full = sbase + kOffBar;                       // [kRawStages]
  const uint32_t bar_raw_empty = bar_raw_full + 8 * kRawStages;        // [kRawStages]
  const uint32_t bar_op_full = bar_raw_empty + 8 * kRawStages;         // [kOpStages]
  const uint32_t bar_op_empty = bar_op_full + 8 * kOpStages;           // [kOpStages]
  float* shift_s = reinterpret_cast<float*>(smem + kOffShift);

  // contiguous tile range of this CTA
  const int64_t total_tiles = (n_rows + kTcRows - 1) / kTcRows;
  const int64_t tile_begin = (int64_t)blockIdx.x * total_tiles / gridDim.x;
  const int64_t tile_end = (int64_t)(blockIdx.x + 1) * total_tiles / gridDim.x;
  const int my_tiles = (int)(tile_end - tile_begin);

  // ---- one-time setup --------------------------------------------------------------------
  if (threadIdx.x == 0) {
    for (int s = 0; s < kRawStages; ++s) {
      mbar_init(bar_raw_full + 8 * s, 1);
      mbar_init(bar_raw_empty + 8 * s, kProducers + (RAWB ? kConsumerWarps : 0));
    }
    for (int s = 0; s < kOpStages; ++s) {
      mbar_init(bar_op_full + 8 * s, kProducers);
      mbar_init(bar_op_empty + 8 * s, kConsumerWarps);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (warp == kTmaWarp && lane == 0) {
    tma_prefetch_desc(&tmX);
    tma_prefetch_desc(&tmY);
    if (has_mask) tma_prefetch_desc(&tmM);
  }
  // zero the operand stages once: feature rows >= d, the unused E rows and the lo/hi padding read as 0
  for (uint32_t o = threadIdx.x * 16; o < kOpStages * kOpStageBytes; o += kThreads * 16)
    *reinterpret_cast<uint4*>(smem + kOffOp + o) = make_uint4(0, 0, 0, 0);
  // packed rows (pack > 1): super-row feature i < pack * d_orig is original feature i % d_orig -> the shift repeats;
  // the columns from pack * d_orig to 127 are TMA out-of-bounds zero fill and keep shift 0 (they contribute nothing)
  for (int j = threadIdx.x; j <= kMaxD; j += kThreads)
    shift_s[j] = (j == kMaxD) ? shift_value(shift, kMaxD, n_shift)
                              : (j < pack * d_orig ? shift_value(shift, j % d_orig, n_shift) : 0.f);
  fence_proxy_async_smem();
  __syncthreads();

  // ---- warp roles --------------------------------------------------------------------------
  if (warp < kConsumerWarps) {
    // ===== consumers: wgmma into register accumulators, fp64 drain to the CTA's partial in global =====
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kConsumerRegs));
    const int wg = warp >> 2;
    if constexpr (RAWB) {
    // fragment of this thread: register 4j + 2h + e holds row (feature) 64 wg + 16 (warp % 4) + lane / 4 + 8 h,
    // column 8 j + 2 (lane % 4) + e, in accX (columns = the 128 raw features) and in accE (columns = E); accX2 / accE2: lo
    float accX[64], accE[8], accX2[64], accE2[8];
    double* my_part = part + (size_t)blockIdx.x * kTcAccElems + 64 * wg + 16 * (warp & 3) + (lane >> 2);
    const int col0 = 2 * (lane & 3);
    const uint32_t a_off = (uint32_t)wg * 8 * kOpSBO;
    int os = 0, held = -1, in_chunk = 0;                   // held: the tile whose stages wait for their MMAs
    uint32_t oph = 0;
    bool first_chunk = true;
    for (int it = 0; it < my_tiles; ++it) {
      mbar_wait(bar_op_full + 8 * os, oph, wait_ns);
      const uint32_t op_addr = sbase + kOffOp + os * kOpStageBytes;
      const uint32_t raw_addr = sbase + kOffRaw + (uint32_t)(it % kRawStages) * kRawStageBytes;
      wgmma_fence();
#pragma unroll
      for (int k2 = 0; k2 < kTcRows / 16; ++k2) {
        const uint32_t k_addr = op_addr + k2 * 2 * kOpLBO;
        const uint64_t x_desc = make_raw_desc(raw_addr + k2 * 16 * 128);        // rows 16 k2 .. 16 k2 + 15
        const uint64_t e_desc = make_smem_desc(k_addr + kOpEOff);
        const uint64_t hi_desc = make_smem_desc(k_addr + a_off);
        const uint32_t sc = (in_chunk > 0 || k2 > 0) ? 1u : 0u;
        wgmma_m64n128k16_bmn(accX, hi_desc, x_desc, sc);
        wgmma_m64n16k16(accE, hi_desc, e_desc, sc);
        if constexpr (SPLIT) {
          const uint64_t lo_desc = make_smem_desc(k_addr + kOpLoOff + a_off);
          const uint32_t sc2 = (it > 0 || k2 > 0) ? 1u : 0u;
          wgmma_m64n128k16_bmn(accX2, lo_desc, x_desc, sc2);
          wgmma_m64n16k16(accE2, lo_desc, e_desc, sc2);
        }
      }
      wgmma_commit();
      const bool last = (in_chunk == chunk_tiles - 1) || (it == my_tiles - 1);
      if (last) {
        wgmma_wait<0>();
        fence_regs(accX);
        fence_regs(accE);
      } else {
        wgmma_wait<1>();
      }
      if (lane == 0) {
        if (held >= 0) {
          mbar_arrive(bar_op_empty + 8 * (held % kOpStages));
          mbar_arrive(bar_raw_empty + 8 * (held % kRawStages));
        }
        if (last) {
          mbar_arrive(bar_op_empty + 8 * os);
          mbar_arrive(bar_raw_empty + 8 * (it % kRawStages));
        }
      }
      held = last ? -1 : it;
      if (last) {
        // sum_r hi_i x_j - c_j sum_r hi_i = sum_r hi_i v_j; sum_r hi_i is E1's ones column, held by lane 4 * (lane / 4)
        const double s1a = (double)__shfl_sync(0xffffffffu, accE[0], lane & ~3);
        const double s1b = (double)__shfl_sync(0xffffffffu, accE[2], lane & ~3);
#pragma unroll
        for (int r = 0; r < 64; ++r) {
          const int col = 8 * (r >> 2) + col0 + (r & 1);
          const double val = (double)accX[r] - (double)shift_s[col] * (((r >> 1) & 1) ? s1b : s1a);
          double* dst = my_part + (size_t)col * kTcM + 8 * ((r >> 1) & 1);
          if (first_chunk) *dst = val;
          else *dst += val;
        }
#pragma unroll
        for (int r = 0; r < 8; ++r) {
          double* dst = my_part + (size_t)(kMaxD + 8 * (r >> 2) + col0 + (r & 1)) * kTcM + 8 * ((r >> 1) & 1);
          if (first_chunk) *dst = (double)accE[r];
          else *dst += (double)accE[r];
        }
        first_chunk = false;
        in_chunk = 0;
      } else {
        ++in_chunk;
      }
      if (++os == kOpStages) { os = 0; oph ^= 1; }
    }
    wgmma_wait<0>();
    double* my_part2 = my_part + (size_t)kTcN * kTcM;      // partial columns [144, 288)
    if constexpr (SPLIT) {
      fence_regs(accX2);
      fence_regs(accE2);
      const double s1a = (double)__shfl_sync(0xffffffffu, accE2[0], lane & ~3);
      const double s1b = (double)__shfl_sync(0xffffffffu, accE2[2], lane & ~3);
#pragma unroll
      for (int r = 0; r < 64; ++r) {
        const int col = 8 * (r >> 2) + col0 + (r & 1);
        my_part2[(size_t)col * kTcM + 8 * ((r >> 1) & 1)] =
            0.5 * ((double)accX2[r] - (double)shift_s[col] * (((r >> 1) & 1) ? s1b : s1a));
      }
#pragma unroll
      for (int r = 0; r < 8; ++r)
        my_part2[(size_t)(kMaxD + 8 * (r >> 2) + col0 + (r & 1)) * kTcM + 8 * ((r >> 1) & 1)] = (double)accE2[r];
    } else {
#pragma unroll
      for (int r = 0; r < kAccRegs; ++r)
        my_part2[(size_t)(8 * (r >> 2) + col0 + (r & 1)) * kTcM + 8 * ((r >> 1) & 1)] = 0.0;
    }
    } else {
    // no plain instruction may write the accumulators between wgmma (ptxas would serialise them): a chunk restarts D1,
    // and the first tile starts D2, with scale-d = 0 on its first K step
    float acc1[kAccRegs], acc2[kAccRegs];
    // fragment of this thread: register 4j + 2h + e holds row (feature) 64 wg + 16 (warp % 4) + lane / 4 + 8 h,
    // column 8 j + 2 (lane % 4) + e; the partial is column-major [col][feature]
    double* my_part = part + (size_t)blockIdx.x * kTcAccElems + 64 * wg + 16 * (warp & 3) + (lane >> 2);
    const int col0 = 2 * (lane & 3);
    const uint32_t a_off = (uint32_t)wg * 8 * kOpSBO;      // this warpgroup's 64 features of A
    int os = 0, held = -1, in_chunk = 0;
    uint32_t oph = 0;
    bool first_chunk = true;
    for (int it = 0; it < my_tiles; ++it) {
      mbar_wait(bar_op_full + 8 * os, oph, wait_ns);
      const uint32_t op_addr = sbase + kOffOp + os * kOpStageBytes;
      wgmma_fence();
#pragma unroll
      for (int k2 = 0; k2 < kTcRows / 16; ++k2) {
        const uint32_t k_addr = op_addr + k2 * 2 * kOpLBO;
        const uint64_t b_desc = make_smem_desc(k_addr);                        // [hi | E]
        if (!(dbg & 2u))                                                                        // A = hi
          wgmma_m64n144k16(acc1, make_smem_desc(k_addr + a_off), b_desc, (in_chunk > 0 || k2 > 0) ? 1u : 0u);
        if (SPLIT && !(dbg & 3u))                                                               // A = lo
          wgmma_m64n144k16(acc2, make_smem_desc(k_addr + kOpLoOff + a_off), b_desc, (it > 0 || k2 > 0) ? 1u : 0u);
      }
      wgmma_commit();
      const bool last = (in_chunk == chunk_tiles - 1) || (it == my_tiles - 1);
      // the previous tile's MMAs are complete after wait_group 1 (this tile's too after wait_group 0): free their stages;
      // the last tile of the range is always `last`, so the accumulators are settled when the loop ends
      if (last) {
        wgmma_wait<0>();
        fence_regs(acc1);
        if constexpr (SPLIT) fence_regs(acc2);
      } else {
        wgmma_wait<1>();
      }
      if (lane == 0) {
        if (held >= 0) mbar_arrive(bar_op_empty + 8 * held);
        if (last) mbar_arrive(bar_op_empty + 8 * os);
      }
      held = last ? -1 : os;
      if (last) {
        // D1 of this chunk: fold into partial columns [0, 144)
#pragma unroll
        for (int r = 0; r < kAccRegs; ++r) {
          double* dst = my_part + (size_t)(8 * (r >> 2) + col0 + (r & 1)) * kTcM + 8 * ((r >> 1) & 1);
          if (first_chunk) *dst = (double)acc1[r];
          else *dst += (double)acc1[r];
        }
        first_chunk = false;
        in_chunk = 0;
      } else {
        ++in_chunk;
      }
      if (++os == kOpStages) { os = 0; oph ^= 1; }
    }
    wgmma_wait<0>();     // a no-op at run time (see above), but ptxas cannot prove it and would wait inside the loop
    if constexpr (SPLIT) fence_regs(acc2);
    // D2 (A = lo) accumulated over the whole range (small zero-mean sums): partial columns [144, 288)
#pragma unroll
    for (int r = 0; r < kAccRegs; ++r)
      my_part[(size_t)(kTcN + 8 * (r >> 2) + col0 + (r & 1)) * kTcM + 8 * ((r >> 1) & 1)] = SPLIT ? (double)acc2[r] : 0.0;
    }
  } else {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kProducerRegs));
    if (warp == kTmaWarp) {
      // ===== TMA producer =====
      if (lane == 0) {
        const uint32_t tx = (uint32_t)(kTcRows * d * sizeof(T)) + kTcRows * pack * 4 + (has_mask ? kTcRows * pack : 0);
        int s = 0;
        uint32_t ph = 0;
        for (int it = 0; it < my_tiles; ++it) {
          mbar_wait(bar_raw_empty + 8 * s, ph ^ 1, wait_ns);
          const uint32_t full = bar_raw_full + 8 * s;
          mbar_expect_tx(full, tx);
          const int64_t row0 = (tile_begin + it) * kTcRows;
          tma_load_2d(sbase + kOffRaw + s * kRawStageBytes, &tmX, 0, (int)row0, full);
          if constexpr (RAWB) tma_load_2d(sbase + kOffRaw + s * kRawStageBytes + kRawBoxBytes, &tmX, 64, (int)row0, full);
          const int sub0 = (int)row0 * pack;                               // first original row of the tile
          if (y_map_2d) tma_load_2d(sbase + kOffY + s * kYStageBytes, &tmY, 0, sub0 >> 2, full);
          else tma_load_1d(sbase + kOffY + s * kYStageBytes, &tmY, sub0, full);
          if (has_mask == 2) tma_load_2d(sbase + kOffMask + s * kMStageBytes, &tmM, 0, sub0 >> 4, full);
          else if (has_mask) tma_load_1d(sbase + kOffMask + s * kMStageBytes, &tmM, sub0, full);
          if (++s == kRawStages) { s = 0; ph ^= 1; }
        }
      }
    } else if (warp == kEWarp) {
      // ===== E warp: extra operand columns [1, y'_hi, y'_lo] and the CUDA-core sums of y' =====
      const float c_y = shift_s[kMaxD];
      double sy = 0.0, syy = 0.0, cnt = 0.0;
      int rs = 0, os = 0;
      uint32_t rph = 0, oph = 0;
      for (int it = 0; it < my_tiles; ++it) {
        mbar_wait(bar_raw_full + 8 * rs, rph, wait_ns);
        mbar_wait(bar_op_empty + 8 * os, oph ^ 1, wait_ns);
        const int64_t row0 = (tile_begin + it) * kTcRows;
        const uint32_t y_addr = sbase + kOffY + rs * kYStageBytes;
        const uint32_t m_addr = sbase + kOffMask + rs * kMStageBytes;
        const uint32_t e_addr = sbase + kOffOp + os * kOpStageBytes + kOpEOff;
        const int64_t left = n_rows - row0;
        const int rows_valid = left < kTcRows ? (int)left : kTcRows;
        float a = 0.f, b = 0.f, c = 0.f;
        for (int half = 0; half < kTcRows / 32; ++half) {   // one super-row per lane and half
          const int rr = lane + 32 * half;                  // super-row inside the tile
          const uint32_t dst = e_addr + (rr >> 3) * kOpLBO + (rr & 7) * 2;
          for (int bl = 0; bl < pack; ++bl) {               // original row rr * pack + bl -> E columns 3*bl .. 3*bl+2
            const int sub = rr * pack + bl;
            bool use = rr < rows_valid;
            if (use && has_mask) use = (ld_shared_u8(m_addr + sub) == (uint32_t)keep);
            const float yv = use ? ld_shared_f32(y_addr + sub * 4) - c_y : 0.f;
            uint32_t yh, yl;
            split2(yv, 0.f, yh, yl);
            st_shared_u16(dst + (3 * bl) * 16, use ? 0x3F80u : 0u);   // bf16(1.0): row-validity ("ones") column
            st_shared_u16(dst + (3 * bl + 1) * 16, yh);
            st_shared_u16(dst + (3 * bl + 2) * 16, yl);
            if (RAWB && has_mask && !use) {         // the raw row is a B operand: clear it (both boxes)
              const uint32_t row = sbase + kOffRaw + rs * kRawStageBytes + (uint32_t)rr * 128;
              const uint32_t z[4] = {0u, 0u, 0u, 0u};
#pragma unroll
              for (int q = 0; q < 8; ++q) { st_shared_v4(row + 16 * q, z); st_shared_v4(row + kRawBoxBytes + 16 * q, z); }
            }
            a += yv;
            b = fmaf(yv, yv, b);
            c += use ? 1.f : 0.f;
          }
        }
        sy += (double)a; syy += (double)b; cnt += (double)c;
        fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) {
          mbar_arrive(bar_op_full + 8 * os);
          mbar_arrive(bar_raw_empty + 8 * rs);
        }
        if (++rs == kRawStages) { rs = 0; rph ^= 1; }
        if (++os == kOpStages) { os = 0; oph ^= 1; }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        sy += __shfl_xor_sync(0xffffffffu, sy, o);
        syy += __shfl_xor_sync(0xffffffffu, syy, o);
        cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
      }
      if (lane == 0) {
        double* ys = side + (size_t)blockIdx.x * kTcSideDoubles;
        ys[0] = sy; ys[1] = syy; ys[2] = cnt;
        ys[3] = 0.0; ys[4] = 0.0; ys[5] = 0.0;
      }
    } else {
      // ===== transform: shift, bf16 hi/lo split, K-major operand store =====
      // A task = (feature quad q of 32 features, 8-row group g) of a tile: nq * 8 tasks per tile over the transform warps.
      const int t = warp - kFirstXformWarp;
      const int nq = (d + 31) >> 5;
      const int n_tasks = nq * kKGroups;
      const uint32_t esz = sizeof(T);
      const uint32_t pitch = (uint32_t)d * esz;       // raw tile row pitch in bytes
      int rs = 0, os = 0;
      uint32_t rph = 0, oph = 0;
      for (int it = 0; it < my_tiles; ++it) {
        mbar_wait(bar_raw_full + 8 * rs, rph, wait_ns);
        mbar_wait(bar_op_empty + 8 * os, oph ^ 1, wait_ns);
        const int64_t row0 = (tile_begin + it) * kTcRows;
        const int64_t left = n_rows - row0;
        const int rows_valid = left < kTcRows ? (int)left : kTcRows;
        const bool full_tile = (!has_mask) && (rows_valid == kTcRows);
        const uint32_t raw_addr = sbase + kOffRaw + rs * kRawStageBytes;
        const uint32_t m_addr = sbase + kOffMask + rs * kMStageBytes;
        const uint32_t op_addr = sbase + kOffOp + os * kOpStageBytes;
        for (int tt = t; tt < n_tasks; tt += kXformWarps) {
          const int q = tt % nq, g = tt / nq;
          const int i = q * 32 + lane;
          if (i < d) {
            const int r0 = g * 8;
            float v[8];
            const uint32_t src = raw_addr + (uint32_t)r0 * pitch + (uint32_t)i * esz;
            const float c_i = shift_s[i];
#pragma unroll
            for (int k = 0; k < 8; ++k) {
              // RAWB: feature i of row r0 + k sits in box i / 64, 16-byte chunk ((i % 64) / 8) ^ k of the 128-byte row
              const uint32_t a = RAWB ? raw_addr + (uint32_t)(i >> 6) * kRawBoxBytes + (uint32_t)(r0 + k) * 128 +
                                            ((((uint32_t)(i & 63) >> 3) ^ (uint32_t)k) << 4) + (uint32_t)(i & 7) * 2
                                      : src + (uint32_t)k * pitch;
              v[k] = ((dbg & 8u) ? __uint_as_float(src + k) : raw_ld_shared<T>(a)) - c_i;
            }
            if (!full_tile) {
              const int blk = i / d_orig;                   // which original row of the super-row this feature belongs to
#pragma unroll
              for (int k = 0; k < 8; ++k) {
                bool use = (r0 + k) < rows_valid;
                if (use && has_mask) use = (ld_shared_u8(m_addr + (r0 + k) * pack + blk) == (uint32_t)keep);
                if (!use) v[k] = 0.f;
              }
            }
            uint32_t hp[4], lp[4];
#pragma unroll
            for (int p = 0; p < 4; ++p) {
              if constexpr (SPLIT) {
                split2(v[2 * p], v[2 * p + 1], hp[p], lp[p]);
              } else {
                const __nv_bfloat162 h = __floats2bfloat162_rn(v[2 * p], v[2 * p + 1]);
                hp[p] = *reinterpret_cast<const uint32_t*>(&h);
                lp[p] = 0u;
              }
            }
            if (!(dbg & 4u)) {
              const uint32_t dst = op_addr + (uint32_t)g * kOpLBO + (uint32_t)((i >> 3) * kOpSBO + (i & 7) * 16);
              st_shared_v4(dst, hp);
              if constexpr (SPLIT) st_shared_v4(dst + kOpLoOff, lp);
            }
          }
        }
        if (!(dbg & 32u)) fence_proxy_async_smem();  // generic-proxy stores -> visible to the tensor core (async proxy)
        __syncwarp();
        if (lane == 0) {
          mbar_arrive(bar_op_full + 8 * os);
          mbar_arrive(bar_raw_empty + 8 * rs);
        }
        if (++rs == kRawStages) { rs = 0; rph ^= 1; }
        if (++os == kOpStages) { os = 0; oph ^= 1; }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// finalize: tc_reduce_kernel sums the per-CTA partials in CTA order (deterministic)
//   red[col * 128 + i], col in [0, 288):  col < 144: D1 (A = hi), col >= 144: D2 (A = lo), columns of [hi | E]
//   red[kTcAccElems + 0..2]            : sum y', sum y'^2, rows used
// tc_fold_kernel undoes the shift in fp64 and adds the result into the raw statistic S ((d+2)^2, stride d+2).
// ------------------------------------------------------------------------------------------

// What tc_finalize_kernel does after the reduce + fold (passed by value).
struct TcFinal {
  int assign;                 // S = value instead of S += value (fresh statistic: no memset launch)
  int n_ranks, rank;          // n_ranks > 1: store S into the exchange slot of every rank and publish the flags
  unsigned int epoch;
  PeerPtrs peers;
};

// ONE launch behind the Gram kernel: reduce the per-CTA partials (fixed order: deterministic), grid barrier, undo the
// shift in fp64 and fold into S, store S into the peers' exchange slots (b2_fit with an attached peer exchange), and
// -- through a last-block ticket -- publish the exchange flags and re-arm the barrier.  Cooperative launch: every CTA
// is resident, so the counter barrier is safe.  This work deliberately does NOT live in the Gram kernel's tail: with
// it there the hot role loops carry its registers and
// code; a separate launch keeps them lean.
constexpr int kFinalizeThreads = 1024;                           // 4 threads per element of the partials
constexpr int kFinalizeCtas = (kRedElems + kFinalizeThreads / 4 - 1) / (kFinalizeThreads / 4);   // 145: one pass

__global__ void __launch_bounds__(kFinalizeThreads, 1)
tc_finalize_kernel(const double* part, const double* side, int n_ctas, double* red, const float* __restrict__ shift,
                   int64_t n_rows, int d, int pack, double* S, unsigned int* sync, const TcFinal fin) {
  __shared__ double quarter[kFinalizeThreads];
  __shared__ double c_s[kMaxD + 1];                              // the shift as fp64 (c_s[kMaxD]: c_y)
  __shared__ float c_part[kShiftBlocks * kShiftStride];          // the 64 partial sums of the shift sample (33 KB)
  // the same values shift_value() gives the Gram kernel -- same operands, same order of the 64 additions -- but with
  // all loads of the CTA in flight at once: the serial walk (8 batches of dependent-latency loads by 129 threads while
  // 895 wait at the next barrier) dominated this kernel
  for (int idx = threadIdx.x; idx < kShiftBlocks * kShiftStride; idx += blockDim.x) c_part[idx] = __ldg(shift + idx);
  __syncthreads();
  for (int j = threadIdx.x; j <= kMaxD; j += blockDim.x) {
    float acc = 0.f;
#pragma unroll 8
    for (int b = 0; b < kShiftBlocks; ++b) acc += c_part[b * kShiftStride + j];
    c_s[j] = (j < d || j == kMaxD) ? (double)__bfloat162float(__float2bfloat16_rn(acc / (float)shift_samples(n_rows))) : 0.0;
  }
  {
    constexpr int epb = kFinalizeThreads / 4;                    // elements per pass of a CTA
    const int per = (((kRedElems + (int)gridDim.x - 1) / (int)gridDim.x) + epb - 1) / epb * epb;
    const int e0 = (int)blockIdx.x * per;
    const int e1 = e0 + per < kRedElems ? e0 + per : kRedElems;
    if (e0 < kRedElems) tc_reduce_range(part, side, n_ctas, red, e0, e1, quarter);
  }
  grid_barrier(sync + 0);
  {
    const int dp = d + 2;
    const int total = dp * dp;
    const size_t slot = xchg_slot_offset(fin.epoch, fin.rank);
    for (int idx = (int)(blockIdx.x * blockDim.x + threadIdx.x); idx < total; idx += (int)(gridDim.x * blockDim.x)) {
      const double val = tc_fold_value(red, c_s, d, pack, idx);
      const double sv = fin.assign ? val : S[idx] + val;
      S[idx] = sv;
      if (fin.n_ranks > 1) xchg_store_all(fin.peers, fin.n_ranks, slot, idx, sv);
    }
    if (fin.n_ranks > 1) __threadfence_system();
  }
  __syncthreads();
  __shared__ bool last_cta;
  if (threadIdx.x == 0) {
    __threadfence();
    last_cta = (atomicAdd(sync + 2, 1u) == gridDim.x - 1);
    if (last_cta) {                       // every CTA has passed the barrier: re-arm it for the next launch
      sync[0] = 0u; sync[2] = 0u;
      __threadfence();
    }
  }
  __syncthreads();
  if (last_cta && fin.n_ranks > 1) xchg_publish(fin.peers, fin.n_ranks, fin.rank, fin.epoch);
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  if (fn == nullptr) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(p);
  }
  return fn;
}

}  // namespace

bool gram_tc_supported(const void* X, int x_dtype, const float* y, int64_t n, int d, int64_t ldx) {
  const int es = x_dtype == B2_F32 ? 4 : 2;
  if (d < 4 || d > kMaxD) return false;
  if ((d * es) % 16 != 0) return false;
  if ((ldx * es) % 16 != 0) return false;
  if ((reinterpret_cast<uintptr_t>(X) & 15) != 0 || (reinterpret_cast<uintptr_t>(y) & 15) != 0) return false;
  if (n < kTcRows) return false;
  if (n > (int64_t)0x7fffffff) return false;  // TMA coordinates are int32
  return true;
}

// d: inner extent of the (super-)row tensor; d_box: inner extent of the smem tile (> d: the rest is zero fill)
// swz64: the raw tile of the bf16 D = 128 path -- [64 rows][64 features] boxes (128-byte rows) with SWIZZLE_128B
static int encode_maps(PFN_encodeTiled encode, const void* X, int x_dtype, int es, const float* y, int64_t n, int d,
                       int d_box, int64_t ldx, int64_t n_y, int pack, const uint8_t* mask, bool swz64, CUtensorMap* tmX_out,
                       CUtensorMap* tmY_out, CUtensorMap* tmM_out, int* y_map_2d_out, int* m_map_2d_out) {
  const cuuint32_t y_box = (cuuint32_t)(kTcRows * pack);   // original rows per tile
  CUtensorMap& tmX = *tmX_out; CUtensorMap& tmY = *tmY_out; CUtensorMap& tmM = *tmM_out;
  memset(&tmM, 0, sizeof(tmM));
  {
    cuuint64_t dims[2] = {(cuuint64_t)d, (cuuint64_t)n};
    cuuint64_t strides[1] = {(cuuint64_t)ldx * es};
    cuuint32_t box[2] = {(cuuint32_t)(swz64 ? 64 : d_box), (cuuint32_t)kTcRows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = encode(&tmX, x_dtype == B2_F32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16,
                        2, const_cast<void*>(X), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        swz64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
      set_error("cuTensorMapEncodeTiled(X) failed with %d (n=%lld d=%d box=%d ldx=%lld)", (int)r, (long long)n, d, d_box,
                (long long)ldx);
      return B2_E_CUDA;
    }
  }
  int y_map_2d = 0;
  {
    cuuint64_t dims[1] = {(cuuint64_t)n_y};
    cuuint64_t strides[1] = {0};
    cuuint32_t box[1] = {y_box};
    cuuint32_t estr[1] = {1};
    CUresult r = CUDA_ERROR_INVALID_VALUE;
    if (y_box <= 256)
      r = encode(&tmY, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 1, const_cast<float*>(y), dims, strides, box, estr,
                 CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                 CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
      // rank-1 maps refused: view y as [ceil(n/4)][4] (16-byte rows) -- the same bytes land in smem
      cuuint64_t dims2[2] = {4, (cuuint64_t)((n_y + 3) / 4)};
      cuuint64_t strides2[1] = {16};
      cuuint32_t box2[2] = {4, y_box / 4};
      cuuint32_t estr2[2] = {1, 1};
      r = encode(&tmY, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(y), dims2, strides2, box2, estr2,
                 CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                 CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      y_map_2d = 1;
      if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled(y) failed with %d", (int)r);
        return B2_E_CUDA;
      }
    }
  }
  if (mask != nullptr && (reinterpret_cast<uintptr_t>(mask) & 15) != 0) {
    set_error("row_mask must be 16-byte aligned for the tensor-core path");
    return B2_E_ARG;
  }
  int m_map_2d = 0;
  if (mask != nullptr) {
    cuuint64_t dims[1] = {(cuuint64_t)n_y};
    cuuint64_t strides[1] = {0};
    cuuint32_t box[1] = {y_box};
    cuuint32_t estr[1] = {1};
    CUresult r = CUDA_ERROR_INVALID_VALUE;
    if (y_box <= 256)
      r = encode(&tmM, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, const_cast<uint8_t*>(mask), dims, strides, box, estr,
                 CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                 CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS && n_y % 16 == 0) {
      // box extents stop at 256: view the mask as [n/16][16] (16-byte rows) -- the same bytes land in smem
      cuuint64_t dims2[2] = {16, (cuuint64_t)(n_y / 16)};
      cuuint64_t strides2[1] = {16};
      cuuint32_t box2[2] = {16, y_box / 16};
      cuuint32_t estr2[2] = {1, 1};
      r = encode(&tmM, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<uint8_t*>(mask), dims2, strides2, box2, estr2,
                 CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                 CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      m_map_2d = 1;
    }
    if (r != CUDA_SUCCESS) {
      set_error("cuTensorMapEncodeTiled(mask) failed with %d", (int)r);
      return B2_E_CUDA;
    }
  }

  *m_map_2d_out = m_map_2d;
  *y_map_2d_out = y_map_2d;
  return B2_OK;
}

// Row packing rule: how many of the n rows the tensor-core launch covers (the rest, < 80 rows, take the CUDA-core kernel)
int64_t gram_tc_main_rows(int64_t n_in, int d_in, int64_t ldx_in, int* pack_out) {
  int pack = 1;
  if (d_in > 16 && d_in <= 64 && ldx_in == d_in) {
    pack = 128 / d_in;
    if (pack > kMaxPack) pack = kMaxPack;
    if (n_in < (int64_t)2 * kTcRows * pack) pack = 1;
  }
  const int group = pack == 1 ? 1 : (pack == 3 ? 48 : (pack == 5 ? 80 : 16));
  if (pack_out != nullptr) *pack_out = pack;
  return n_in - n_in % group;
}

int launch_gram_tc(b2_ctx* ctx, const void* X, int x_dtype, const float* y, int64_t n_in, int d_in, int64_t ldx_in,
                   const uint8_t* mask, int keep, const TcFuse* fuse) {
  PFN_encodeTiled encode = get_encode();
  if (encode == nullptr) {
    set_error("cuTensorMapEncodeTiled is not available from the driver");
    return B2_E_CUDA;
  }
  const int es = x_dtype == B2_F32 ? 4 : 2;
  // Row packing: `pack` contiguous rows of 17..64 features are viewed as one super-row of pack * d_in <= 128 columns
  // ([n / pack][pack * d_in], zero-filled by TMA to the 128-wide tile) and run on the D = 128 fast path; the diagonal
  // d_in x d_in blocks of the 128 x 128 Gram sum to the true statistic (tc_fold_kernel).  The tensor maps cover a
  // multiple of lcm(pack, 16) rows (the y / mask views are 16-byte rows); the < 80 leftover rows go through the
  // CUDA-core kernel.
  int pack = 1;
  const int64_t n_main = gram_tc_main_rows(n_in, d_in, ldx_in, &pack);   // original rows handled here
  const int64_t n = n_main / pack;                      // super-rows
  const int d = pack > 1 ? 128 : d_in;                  // kernel feature count (DFIX = 128 when packed)
  const int d_tensor = d_in * pack;                     // columns that exist; the tile is zero-filled beyond them
  const int64_t ldx = ldx_in * pack;
  const int64_t n_y = n_main;                           // y / mask elements covered by the tensor maps
  // bf16-stored rows with D = 128: the raw tile is the MMA's B operand (RAWB)
  const bool rawb = x_dtype == B2_BF16 && d_in == 128 && pack == 1;
  CUtensorMap tmX, tmY, tmM;
  int y_map_2d = 0, m_map_2d = 0;
  b2_ctx::TmCache& tc = ctx->tm_cache;
  const bool cached = tc.X == X && tc.y == y && tc.mask == mask && tc.n == n_in && tc.ldx == ldx_in && tc.d == d_in &&
                      tc.x_dtype == x_dtype;
  if (cached) {
    memcpy(&tmX, tc.tmX, sizeof(tmX)); memcpy(&tmY, tc.tmY, sizeof(tmY)); memcpy(&tmM, tc.tmM, sizeof(tmM));
    y_map_2d = tc.y_map_2d & 1; m_map_2d = (tc.y_map_2d >> 1) & 1;
  } else {
    if (int r = encode_maps(encode, X, x_dtype, es, y, n, d_tensor, d, ldx, n_y, pack, mask, rawb, &tmX, &tmY, &tmM, &y_map_2d,
                            &m_map_2d))
      return r;
    tc.X = X; tc.y = y; tc.mask = mask; tc.n = n_in; tc.ldx = ldx_in; tc.d = d_in; tc.x_dtype = x_dtype;
    tc.y_map_2d = y_map_2d | (m_map_2d << 1);
    memcpy(tc.tmX, &tmX, sizeof(tmX)); memcpy(tc.tmY, &tmY, sizeof(tmY)); memcpy(tc.tmM, &tmM, sizeof(tmM));
  }

  const int64_t total_tiles = (n + kTcRows - 1) / kTcRows;
  const int sms = (ctx->sm_limit > 0 && ctx->sm_limit < ctx->sm_count) ? ctx->sm_limit : ctx->sm_count;
  const int grid = (int)(total_tiles < sms ? total_tiles : sms);
  // the RAWB accumulators carry the unshifted x (sum hi_i x_j includes c_j sum hi_i): a quarter of the fp32 chain length
  // keeps their truncation error at the level of the shifted operands' accumulators
  int chunk_tiles = ctx->drain_rows / kTcRows / (rawb ? 4 : 1);
  if (chunk_tiles < 1) chunk_tiles = 1;

  if (!ctx->tc_attr_set) {
#define B2_SET_SMEM(T, DF, SP) \
  B2_CUDA(cudaFuncSetAttribute(gram_tc_kernel<T, DF, SP>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes))
    B2_SET_SMEM(float, 128, true); B2_SET_SMEM(float, 0, true);
    B2_SET_SMEM(float, 128, false); B2_SET_SMEM(float, 0, false);
    B2_SET_SMEM(__nv_bfloat16, 128, true); B2_SET_SMEM(__nv_bfloat16, 0, true);
    B2_SET_SMEM(__nv_bfloat16, 128, false); B2_SET_SMEM(__nv_bfloat16, 0, false);
#undef B2_SET_SMEM
    B2_CUDA(cudaFuncSetAttribute(gram_tc_kernel<__nv_bfloat16, 128, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 kSmemBytes));
    B2_CUDA(cudaFuncSetAttribute(gram_tc_kernel<__nv_bfloat16, 128, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 kSmemBytes));
    ctx->tc_attr_set = true;
  }

  // S: a fresh statistic is overwritten by the finalize kernel (no memset launch); otherwise it must be cleared first
  const bool assign = fuse != nullptr && fuse->assign != 0;
  if (!assign) {
    if (int r = ensure_s_cleared(ctx)) return r;
  }
  if (x_dtype == B2_F32)
    tc_shift_kernel<float><<<kShiftBlocks, kShiftCols * kShiftGroups, 0, ctx->stream>>>(static_cast<const float*>(X), y, n_in, d_in,
                                                                  ldx_in, ctx->shift);
  else
    tc_shift_kernel<__nv_bfloat16><<<kShiftBlocks, kShiftCols * kShiftGroups, 0, ctx->stream>>>(static_cast<const __nv_bfloat16*>(X), y,
                                                                          n_in, d_in, ldx_in, ctx->shift);
  B2_CUDA(cudaGetLastError());

#ifdef B2_DEV_KNOBS
  static const uint32_t wait_ns = []() {   // development knob: suspend-time hint of the pipeline waits
    const char* e = getenv("B2_WAIT_HINT_NS");
    return e ? (uint32_t)atoi(e) : 20000u;
  }();
#else
  constexpr uint32_t wait_ns = 20000u;     // try_wait suspend hint (ns); measured insensitive 0..20000 (r01)
#endif
#ifdef B2_DEV_KNOBS
  static const uint32_t dbg = []() {       // ablations: bit0 skip MMA2, bit1 skip all MMAs, bit2 skip STS, bit3 skip LDS, bit5 skip proxy fence
    const char* e = getenv("B2_TC_DEBUG");
    return e ? (uint32_t)atoi(e) : 0u;
  }();
#else
  constexpr uint32_t dbg = 0u;
#endif
  const int pair = ctx->k_pairs % kKernelEventPairs;
  B2_CUDA(cudaEventRecord(ctx->ev_k[pair][0], ctx->stream));
#define B2_LAUNCH_TC(T, DF, SP, RB)                                                                      \
  gram_tc_kernel<T, DF, SP, RB><<<grid, kThreads, kSmemBytes, ctx->stream>>>(                                \
      tmX, tmY, tmM, y_map_2d, mask != nullptr ? 1 + m_map_2d : 0, keep, n, d, pack, d_in, n_in, ctx->shift, \
      chunk_tiles,                                                                                        \
      ctx->tc_part, ctx->tc_side, wait_ns, dbg)
#define B2_LAUNCH_TC_D(T, SP) \
  do { if (d == 128) B2_LAUNCH_TC(T, 128, SP, false); else B2_LAUNCH_TC(T, 0, SP, false); } while (0)
  const bool split = ctx->precision == B2_PRECISION_SPLIT;
  if (rawb) {
    if (split) B2_LAUNCH_TC(__nv_bfloat16, 128, true, true); else B2_LAUNCH_TC(__nv_bfloat16, 128, false, true);
  } else if (x_dtype == B2_F32) {
    if (split) B2_LAUNCH_TC_D(float, true); else B2_LAUNCH_TC_D(float, false);
  } else {
    if (split) B2_LAUNCH_TC_D(__nv_bfloat16, true); else B2_LAUNCH_TC_D(__nv_bfloat16, false);
  }
#undef B2_LAUNCH_TC_D
#undef B2_LAUNCH_TC
  B2_CUDA(cudaGetLastError());
  B2_CUDA(cudaEventRecord(ctx->ev_k[pair][1], ctx->stream));
  ctx->k_pairs += 1;

  // finalize: reduce + fold (+ peer scatter) in one cooperative launch
  TcFinal fin;
  memset(&fin, 0, sizeof(fin));
  fin.assign = assign ? 1 : 0;
  fin.n_ranks = 1;
  if (fuse != nullptr && fuse->scatter) {
    fin.n_ranks = ctx->n_ranks; fin.rank = ctx->rank; fin.epoch = fuse->epoch;
    for (int r = 0; r < kMaxRanks; ++r) fin.peers.p[r] = ctx->xchg_peer[r];
  }
  {
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3(kFinalizeCtas < sms ? kFinalizeCtas : sms);
    cfg.blockDim = dim3(kFinalizeThreads); cfg.dynamicSmemBytes = 0; cfg.stream = ctx->stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeCooperative;
    attr[0].val.cooperative = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    const double* part_arg = ctx->tc_part; const double* side_arg = ctx->tc_side;
    const float* shift_arg = ctx->shift;
    B2_CUDA(cudaLaunchKernelEx(&cfg, tc_finalize_kernel, part_arg, side_arg, grid, ctx->tc_red, shift_arg, n_in, d_in, pack,
                               ctx->S, ctx->tc_sync, fin));
  }
  ctx->launches += 3;
  ctx->k_launches += 3;
  ctx->s_zero_pending = false;
  const bool fused = fuse != nullptr;
  if (n_main < n_in && !fused) {   // the n % pack leftover rows (the fused caller accumulates them first)
    const char* Xt = static_cast<const char*>(X) + (size_t)n_main * ldx_in * es;
    return launch_gram_simt(ctx, Xt, x_dtype, y + n_main, n_in - n_main, d_in, ldx_in,
                            mask != nullptr ? mask + n_main : nullptr, keep);
  }
  return B2_OK;
}

}  // namespace b2
