// gram_tc.cu -- the hot kernel: row-block streaming Gram accumulator on the Hopper tensor core (wgmma, sm_90a).
//
// Replaces the pass over the training rows inside LinearRegression.fit
// (stage_1_train_model.py:105-106 -> sklearn/linear_model/_base.py: centre + LAPACK gelsd).
//
// Data flow per CTA (persistent, one CTA per SM, contiguous range of 64-row tiles):
//
//   HBM --TMA (cp.async.bulk.tensor, evict-first)--> smem raw tile [64 rows][D] (+ y, + row mask)
//     --8 transform warps (two per SM sub-partition; one lane of one of them also issues the TMA loads):
//        v = x - c (per-column shift), bf16 split v = hi + lo;
//        one of them also writes the extra columns E = [1, y'_hi, y'_lo] (y' = y - c_y), CUDA-core sums of y', y'^2, rows
//     --> operands, K-major canonical layout (8 x 16 B core matrices, no swizzle; one 16-byte chunk =
//         8 consecutive rows of X for one feature), per 8-row K group:
//            rows j = 0..127 hi | 128..143 E | 144..271 lo          (B = [hi | E], A = hi or A = lo)
//     --wgmma.mma_async (bf16 x bf16 -> fp32 in registers); warpgroup c (c = 0, 1) owns features 64c..64c+63 (A side),
//       two wgmma per K step of 16 rows, EW = 8 E columns (16 for rows packed 3 or more to a super-row):
//            D1[i][j] += sum_r hi[r][i] * [hi | E][r][j], j >= 64c   m64n(128 - 64c + EW): hi^T hi is symmetric, so
//                                                                     warpgroup 1 skips the block warpgroup 0 has
//                                                                     transposed; drained every `drain_rows` rows
//            D2[i][j] += sum_r lo[r][i] * [hi | E][r][j]             m64n(128 + EW): small zero-mean terms, drained
//                                                                     once at the end
//        so D1[:, :128] = hi^T hi (i <= j), D2[:, :128] = lo^T hi, column 128 = sum v, columns 129/130 = sum v*y'.
//     --every `drain_rows` rows the two consumer warpgroups add the entries of D1 the fold reads (i <= j, and E) to
//        their running fp64 sums and restart D1 from zero; the producer warps keep filling stages meanwhile.  A sum
//        lives in its owner thread's registers, in a shared-memory slab, or for the entries that fit in neither in
//        this CTA's fp64 partial in global memory (L2-resident; fire-and-forget red.add.f64); the end of the range
//        stores the on-chip sums to the partial (layout: tc_part_index).
//       The accumulator registers (136 or 144 per thread of warpgroup 0) come from the producers (setmaxnreg).
//
// Why the shift and the split: the tensor core accumulates fp32 with truncation, so raw (uncentred)
// second moments cannot reach the 1e-4 coefficient tolerance; after the shift the Gram is ~diagonal and
// the centring in the solve subtracts almost nothing.  hi+lo carries 16 mantissa bits, i.e. products are
// accurate to ~2^-17 relative (lo*lo is dropped).
//
// The shift c comes from gram_shift.cu.  tc_finalize_kernel sums the per-CTA partials in a fixed order
// (deterministic), reading only the entries this launch wrote, undoes the shift in fp64 and adds the result to the
// context's raw statistic S = [X 1 y]^T [X 1 y].
#include <cuda_bf16.h>
#include <stdlib.h>

#include "b2_internal.cuh"
#include "b2_ptx.cuh"
#include "b2_shift.cuh"
#include "b2_xchg.cuh"

namespace b2 {
namespace {

// ------------------------------------------------------------------------------------------
// geometry
// ------------------------------------------------------------------------------------------
constexpr int kConsumerWGs = 2;                    // warpgroups 0-1: wgmma + drain, 64 features each
constexpr int kXformWarps = 8;                     // warpgroups 2-3: transform, two warps on each SM sub-partition
constexpr int kThreads = 128 * (kConsumerWGs + 2); // warps: 0-7 consumers, 8-15 transform
constexpr int kFirstXformWarp = 4 * kConsumerWGs;
constexpr int kTmaWarp = kFirstXformWarp;          // its lane 0 also issues the TMA loads (sub-partition 0)
constexpr int kEWarp = kFirstXformWarp + 1;        // also writes E and sums y' (sub-partition 1)
static_assert(kFirstXformWarp + kXformWarps == kThreads / 32, "warp roles");
constexpr int kProducers = kXformWarps;            // arrivals that fill an operand stage
constexpr int kConsumerWarps = 4 * kConsumerWGs;   // arrivals that free an operand stage
constexpr int kKGroups = kTcRows / 8;              // 8-row K groups per stage
constexpr uint32_t kRawStageBytes = kTcRows * kMaxD * 4;      // 32768 (fp32, D = 128)
constexpr uint32_t kOpSBO = 128;                              // bytes between 8-row j groups (core matrices along M/N)
constexpr uint32_t kOpLBO = (16 + 2 + 16) * kOpSBO;           // 4352: hi | E | lo groups per K group
constexpr uint32_t kOpEOff = 16 * kOpSBO;                     // E block inside a K group
constexpr uint32_t kOpLoOff = 18 * kOpSBO;                    // lo block inside a K group
constexpr uint32_t kOpStageBytes = kKGroups * kOpLBO;         // 34816
constexpr int kMaxPack = 5;                                             // original rows per 128-wide super-row (3 E columns each)
constexpr uint32_t kYStageBytes = kTcRows * kMaxPack * 4;               // 1280
constexpr uint32_t kMStageBytes = 384;                                  // 64 * kMaxPack = 320 mask bytes, padded: TMA
                                                                        // destinations are 128-byte aligned
static_assert(kMStageBytes >= kTcRows * kMaxPack && kMStageBytes % 128 == 0 && kYStageBytes % 128 == 0, "stage alignment");

// Pipeline depth and shared-memory layout of a variant.  The consumers hold operand stage `it` until the MMAs of it + 1
// are issued, so with 3 operand stages the transform of it + 2 overlaps the MMAs of it + 1 instead of waiting for
// those of `it` (3 raw + 3 operand stages: ~205 KB; 4 + 3 does not fit in 227 KB).  RAWB also holds its raw stage
// until its MMAs have read it, so it keeps 4 raw stages (two tiles of prefetch) and 2 operand stages.
template <bool RAWB>
struct TcGeo {
  static constexpr int kRawStages = RAWB ? 4 : 3;
  static constexpr int kOpStages = RAWB ? 2 : 3;
  // tiles the TMA issue (lane 0 of kTmaWarp) runs ahead of its own transform: before converting tile `it` it waits for
  // the raw stage of tile it + kAhead - kRawStages.  The transform warps release tile it - 1 without waiting for this
  // warp; RAWB's consumers release tile k only after the MMAs of k + 1 are issued, which needs this warp's transform of
  // k + 1, so RAWB may wait for tile it - 2 at most.
  static constexpr int kAhead = RAWB ? kRawStages - 2 : kRawStages - 1;
  static constexpr uint32_t kOffRaw = 0;
  static constexpr uint32_t kOffOp = kOffRaw + kRawStages * kRawStageBytes;
  static constexpr uint32_t kOffY = kOffOp + kOpStages * kOpStageBytes;
  static constexpr uint32_t kOffMask = kOffY + kRawStages * kYStageBytes;
  static constexpr uint32_t kOffBar = kOffMask + kRawStages * kMStageBytes;
  static constexpr int kNumBars = 2 * kRawStages + 2 * kOpStages;
  static constexpr uint32_t kOffShift = kOffBar + kNumBars * 8;
  static constexpr uint32_t kOffESum = kOffShift + (kMaxD + 4) * 4;    // kEWarp's per-lane fp64 sums [3][32]
  // the consumers' running fp64 sums of drained D1 entries that live in shared memory (TcSums):
  // [consumer warp 0..3 of warpgroup 0, then of warpgroup 1][slot][lane], conflict-free, the rest of the 227 KB
  static constexpr int kSlabSlots = RAWB ? 22 : 21;                     // per thread, both warpgroups together
  static constexpr uint32_t kOffSlab = kOffESum + 3 * 32 * 8;
  static constexpr uint32_t kSmemBytes = kOffSlab + kSlabSlots * 4 * 32 * 8 + 1024;  // + alignment slack (~227 KB)
  static_assert(kSmemBytes <= 227 * 1024, "shared memory budget");
  // setmaxnreg split of the 64 K-register file (128 x 512 threads): up to 144 fp32 accumulators per consumer thread.  A
  // transform lane holds 16 values of two features and, at runtime d, eight row addresses: 64 registers.  RAWB's
  // consumers also hold the raw-tile descriptors and need 200, which leaves its transform (fixed pitch) 56.
  static constexpr uint32_t kConsumerRegs = RAWB ? 200 : 192, kProducerRegs = RAWB ? 56 : 64;
  static_assert(kConsumerRegs * 128 * kConsumerWGs + kProducerRegs * (kThreads - 128 * kConsumerWGs) <= 65536,
                "register budget");
};

// Where a consumer thread keeps the running fp64 sum of each D1 entry it drains, between the drains of a range:
// the top kRegs of its kR1 D1 registers in `double` registers, the kSlab below them in its slots of the shared slab,
// the rest in the CTA's partial in L2 (red.add.f64).  The top registers hold the E columns and the highest feature
// columns, the ones whose entries are all in the upper triangle.  The budgets are what the accumulators leave of the
// consumers' setmaxnreg registers without spills (-Xptxas -v): warpgroup 1 keeps all its sums in registers, so warpgroup
// 0 takes the whole slab.
template <int DFIX, bool SPLIT, bool RAWB, int EW, int WG>
struct TcSums {
  static constexpr int kR1 = (kTcM - 64 * WG + EW) / 2;
  static constexpr bool kTight = SPLIT && !RAWB && (EW == 16 || DFIX == 0);
  static constexpr int kRegs = WG == 1 ? (kTight ? (EW == 16 ? 24 : 28) : kR1)
                                       : (!SPLIT ? 40 : (RAWB || EW == 16 ? 0 : (DFIX ? 16 : 8)));
  static constexpr int kSlab = WG == 1 ? 0 : TcGeo<RAWB>::kSlabSlots;
  static constexpr int kSlabBase = WG == 1 ? TcSums<DFIX, SPLIT, RAWB, EW, 0>::kSlab : 0;   // slots of warpgroup 0 before
  static constexpr int kFirstSlab = kR1 - kRegs - kSlab, kFirstReg = kR1 - kRegs;      // register index ranges
  static_assert(kFirstSlab >= 0 && kSlabBase + kSlab <= TcGeo<RAWB>::kSlabSlots, "fp64 sum homes");
};

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
// D[64 x N] (+)= A[64 x 16] * B[16 x N]: bf16 operands from shared memory, A K-major; B K-major (TB = 0) or MN-major
// (TB = 1: the raw 128B-swizzled TMA tile).  fp32 accumulators d[0 .. N/2) in registers (wgmma fragment layout);
// scale_d = 0 overwrites D.  Issued by all 128 threads of a warpgroup.
template <int N, int TB>
__device__ __forceinline__ void wgmma(float* d, uint64_t adesc, uint64_t bdesc, uint32_t scale_d);
#define B2_ACC4(o) "+f"(d[o]), "+f"(d[o + 1]), "+f"(d[o + 2]), "+f"(d[o + 3])
#define B2_ACC8(o) B2_ACC4(o), B2_ACC4(o + 4)
template <>
__device__ __forceinline__ void wgmma<8, 0>(float* d, uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %6, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n8k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3}, "
      "%4, %5, p, 1, 1, 0, 0;\n\t}"
      : B2_ACC4(0)
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
}
template <>
__device__ __forceinline__ void wgmma<72, 0>(float* d, uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %38, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n72k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35}, "
      "%36, %37, p, 1, 1, 0, 0;\n\t}"
      : B2_ACC8(0), B2_ACC8(8), B2_ACC8(16), B2_ACC8(24), B2_ACC4(32)
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
}
template <>
__device__ __forceinline__ void wgmma<80, 0>(float* d, uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %42, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n80k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39}, "
      "%40, %41, p, 1, 1, 0, 0;\n\t}"
      : B2_ACC8(0), B2_ACC8(8), B2_ACC8(16), B2_ACC8(24), B2_ACC8(32)
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
}
template <>
__device__ __forceinline__ void wgmma<136, 0>(float* d, uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %70, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n136k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
      "%64, %65, %66, %67}, "
      "%68, %69, p, 1, 1, 0, 0;\n\t}"
      : B2_ACC8(0), B2_ACC8(8), B2_ACC8(16), B2_ACC8(24), B2_ACC8(32), B2_ACC8(40), B2_ACC8(48), B2_ACC8(56), B2_ACC4(64)
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
}
template <>
__device__ __forceinline__ void wgmma<144, 0>(float* d, uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %74, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n144k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
      "%64, %65, %66, %67, %68, %69, %70, %71}, "
      "%72, %73, p, 1, 1, 0, 0;\n\t}"
      : B2_ACC8(0), B2_ACC8(8), B2_ACC8(16), B2_ACC8(24), B2_ACC8(32), B2_ACC8(40), B2_ACC8(48), B2_ACC8(56), B2_ACC8(64)
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
}
template <>
__device__ __forceinline__ void wgmma<64, 1>(float* d, uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "%32, %33, p, 1, 1, 0, 1;\n\t}"
      : B2_ACC8(0), B2_ACC8(8), B2_ACC8(16), B2_ACC8(24)
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
}
template <>
__device__ __forceinline__ void wgmma<128, 1>(float* d, uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, 0, 1;\n\t}"
      : B2_ACC8(0), B2_ACC8(8), B2_ACC8(16), B2_ACC8(24), B2_ACC8(32), B2_ACC8(40), B2_ACC8(48), B2_ACC8(56)
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
}
#undef B2_ACC8
#undef B2_ACC4
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
__device__ __forceinline__ uint32_t lane_id() {   // volatile: re-read where used instead of kept in a register
  uint32_t l;
  asm volatile("mov.u32 %0, %%laneid;" : "=r"(l));
  return l;
}
__device__ __forceinline__ void st_shared_f64(uint32_t addr, double v) {
  asm volatile("st.shared.f64 [%0], %1;" ::"r"(addr), "d"(v) : "memory");
}
__device__ __forceinline__ double ld_shared_f64(uint32_t addr) {
  double v;
  asm volatile("ld.shared.f64 %0, [%1];" : "=d"(v) : "r"(addr) : "memory");
  return v;
}
// *p += v (add, a fire-and-forget reduction in L2) or *p = v, where `on`: a predicated instruction, not a branch -- a
// divergent path around the registers wgmma owns makes ptxas serialise the wgmma
__device__ __forceinline__ void put_f64(double* p, double v, bool add, bool on) {
  if (add)
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %2, 0;\n\t@p red.global.add.f64 [%0], %1;\n\t}"
                 ::"l"(p), "d"(v), "r"((uint32_t)on) : "memory");
  else
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %2, 0;\n\t@p st.global.f64 [%0], %1;\n\t}"
                 ::"l"(p), "d"(v), "r"((uint32_t)on) : "memory");
}
__device__ __forceinline__ void st_shared_f64_if(uint32_t addr, double v, bool on) {   // predicated, as put_f64
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %2, 0;\n\t@p st.shared.f64 [%0], %1;\n\t}"
               ::"r"(addr), "d"(v), "r"((uint32_t)on) : "memory");
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
// finalize: the per-CTA partials reduced into
//   red[0 .. n_acc)                    : the accumulator entries a launch writes (tc_part_index, b2_internal.cuh)
//   red[kTcAccElems + 0..2]            : sum y', sum y'^2, rows used (the E warp's CUDA-core sums)
// Entry idx < n_acc of CTA c of an n_ctas grid sits at part[c * kTcAccElems + idx]; sum s at
// part[n_ctas * kTcAccElems + c * kTcSums + s] (behind all accumulators, so that every CTA's accumulators keep the
// kTcAccElems stride).  Entries from n_acc to kTcAccElems were not written by this launch and are never read.
// ------------------------------------------------------------------------------------------
constexpr int kRedElems = kTcAccElems + kTcSums;   // the most elements a reduce covers

// Sum over the CTAs of elements [e0, e1) of the n_acc + kTcSums written elements: element idx < n_acc is accumulator
// entry idx, element n_acc + s is sum s.  4 threads per element: thread (e, q) sums the q-th quarter of the CTAs with
// 8 loads in flight (the loads are the latency: a serial walk over the CTAs costs one L2 round trip each, ~140 ns per
// CTA), the quarters are combined in the fixed order 0..3 -> deterministic.  `quarter`: shared scratch of
// 4 * (blockDim.x / 4) doubles.  Call with the whole block.
__device__ __forceinline__ void tc_reduce_range(const double* part, int n_ctas, int n_acc, double* red, int e0, int e1,
                                                double* quarter) {
  const int epb = blockDim.x >> 2;                 // elements per pass
  const int e = threadIdx.x % epb, q = threadIdx.x / epb;
  const int per = (n_ctas + 3) / 4;
  const int c0 = q * per, c1 = (c0 + per < n_ctas) ? c0 + per : n_ctas;
  for (int base = e0; base < e1; base += epb) {
    const int idx = base + e;
    const bool sum = idx >= n_acc;
    if (idx < e1) {
      const double* src = sum ? part + (size_t)n_ctas * kTcAccElems + (idx - n_acc) : part + idx;
      const size_t stride = sum ? kTcSums : kTcAccElems;                        // from one CTA to the next
      double acc[8] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
      int c = c0;
      for (; c + 8 <= c1; c += 8) {
#pragma unroll
        for (int u = 0; u < 8; ++u) acc[u] += __ldcg(src + (size_t)(c + u) * stride);
      }
      for (; c < c1; ++c) acc[0] += __ldcg(src + (size_t)c * stride);
      quarter[q * epb + e] = ((acc[0] + acc[1]) + (acc[2] + acc[3])) + ((acc[4] + acc[5]) + (acc[6] + acc[7]));
    }
    __syncthreads();
    if (q == 0 && idx < e1)
      red[sum ? kTcAccElems + (idx - n_acc) : idx] =
          ((quarter[e] + quarter[epb + e]) + quarter[2 * epb + e]) + quarter[3 * epb + e];
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
// Returns the contribution of this launch to S[idx]; c[j] = the shift of feature j, c[kMaxD] = the shift of y.
// ew: the E columns of the launch; d2: it wrote D2 (hi + lo operands without RAWB), whose lo^T hi terms enter in both
// orientations.  Otherwise D1 already holds sum v_a v_b for a <= b (one operand, or RAWB with lo added in).
__device__ __forceinline__ double tc_fold_value(const double* red, const double* c, int d, int pack, int ew, bool d2,
                                                int idx) {
  const int dp = d + 2;
  const int a = min(idx / dp, idx % dp), b = max(idx / dp, idx % dp);
  auto P = [&](int acc, int i, int j) { return __ldcg(red + tc_part_index(acc, i, j, ew)); };
  auto s1 = [&](int i) {                                                     // sum (x_i - c_i)
    double t = 0.0;
    for (int blk = 0; blk < pack; ++blk) {
      const int r = blk * d + i, e = kTcM + 3 * blk;
      t += d2 ? P(0, r, e) + P(1, r, e) : P(0, r, e);
    }
    return t;
  };
  auto sxy = [&](int i) {                                                    // sum (x_i - c_i) y'
    double t = 0.0;
    for (int blk = 0; blk < pack; ++blk) {
      const int r = blk * d + i, e = kTcM + 3 * blk;
      t += d2 ? P(0, r, e + 1) + P(0, r, e + 2) + P(1, r, e + 1) + P(1, r, e + 2) : P(0, r, e + 1) + P(0, r, e + 2);
    }
    return t;
  };
  auto G = [&](int i, int j) {                    // sum v_i v_j ~= hi.hi + lo.hi + hi.lo   (lo.lo dropped, ~2^-18 relative)
    double g = 0.0;
    for (int blk = 0; blk < pack; ++blk) {
      const int ia = blk * d + i, ib = blk * d + j;
      const double g1 = P(0, min(ia, ib), max(ia, ib));
      g += d2 ? g1 + P(1, ia, ib) + P(1, ib, ia) : g1;
    }
    return g;
  };
  return unshift_entry(a, b, d, c, G, s1, sxy, __ldcg(red + kTcAccElems + 2), __ldcg(red + kTcAccElems + 0),
                       __ldcg(red + kTcAccElems + 1));
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
//   lo has its own accumulators (small zero-mean sums); since the B side is the exact v, sum v_a v_b = sum hi_a v_b +
//   sum lo_a v_b for a <= b, so the end of the range adds them, unhalved, into the same D1 entries and writes no D2.
//   The raw stage is held until the MMAs have read it; masked-out rows are zeroed in it (0 * NaN would poison the sums).
// EW: the E columns the MMAs cover (tc_e_width: 8 up to pack = 2, 16 beyond; runtime-d kernels are unpacked).
template <typename T, int DFIX, bool SPLIT, bool RAWB = false, int EW = 8>
__global__ void __launch_bounds__(kThreads, 1)
gram_tc_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmY,
               const __grid_constant__ CUtensorMap tmM, int y_map_2d, int has_mask, int keep,
               int64_t n_rows, int d_arg, int pack, int d_orig, const float* __restrict__ shift,
               int chunk_tiles, double* __restrict__ part, uint32_t wait_ns, uint32_t dbg_arg) {
#ifdef B2_DEV_KNOBS
  const uint32_t dbg = dbg_arg;      // ablation switches (tools/build_dev.sh): results are WRONG when non-zero, except
                                     // with bit 8 alone
#else
  constexpr uint32_t dbg = 0u;       // product build: the ablation branches compile away
  (void)dbg_arg;
#endif
  using G = TcGeo<RAWB>;
  constexpr int kRawStages = G::kRawStages, kOpStages = G::kOpStages;
  constexpr uint32_t kOffRaw = G::kOffRaw, kOffOp = G::kOffOp, kOffY = G::kOffY, kOffMask = G::kOffMask;
  const int d = DFIX ? DFIX : d_arg;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem = smem_raw + (sbase - smem_u32(smem_raw));
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  const uint32_t bar_raw_full = sbase + G::kOffBar;                    // [kRawStages]
  const uint32_t bar_raw_empty = bar_raw_full + 8 * kRawStages;        // [kRawStages]
  const uint32_t bar_op_full = bar_raw_empty + 8 * kRawStages;         // [kOpStages]
  const uint32_t bar_op_empty = bar_op_full + 8 * kOpStages;           // [kOpStages]
  float* shift_s = reinterpret_cast<float*>(smem + G::kOffShift);

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
    shift_s[j] = j == kMaxD ? shift[kMaxD] : (j < pack * d_orig ? shift[j % d_orig] : 0.f);
  fence_proxy_async_smem();
  __syncthreads();

  // ---- warp roles --------------------------------------------------------------------------
  if (warp < kConsumerWarps) {
    // ===== consumers: wgmma into register accumulators, fp64 drain to the CTA's partial in global =====
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(G::kConsumerRegs));
    // Warpgroup WG owns features 64 WG .. 64 WG + 63 (the A side).  hi^T hi is symmetric, so its D1 covers only the
    // B columns from 64 WG on: [hi rows 64 WG .. 127 | E], kF1 feature columns; in the operand stage those rows and E
    // are contiguous at stride kOpSBO, so the B descriptor starts at the same address as the warpgroup's A.  D2 (A = lo)
    // needs both orientations and covers [hi | E] in full, except with RAWB, whose lo sums enter D1 (see above).
    // One copy of the loop per warpgroup: every wgmma in it has a fixed shape.
    auto consume = [&](auto wg_c) {
      constexpr int WG = decltype(wg_c)::value;
      constexpr int kF1 = kTcM - 64 * WG;                        // D1 feature columns: 64 WG .. 127
      constexpr int kF2 = RAWB ? kF1 : kTcM;                     // D2 feature columns: 64 WG .. 127 or 0 .. 127
      constexpr int kC1 = 64 * WG;                               // D1's partial column of accumulator column 0
      constexpr int kR1 = (kF1 + EW) / 2, kR2 = (kF2 + EW) / 2;  // fp32 accumulator registers per thread
      // no plain instruction may write the accumulators between wgmma (ptxas would serialise them): a chunk restarts D1,
      // and the first tile starts D2, with scale-d = 0 on its first K step
      float acc1[kR1], acc2[kR2];
      // fragment of this thread: register 4j + 2h + e holds row (feature) 64 WG + 16 (warp % 4) + lane / 4 + 8 h,
      // accumulator column 8 j + 2 (lane % 4) + e, partial column col0 + that (an E column from 128 on).
      // store(dst_acc, col0, add, val) writes (or adds) val(r, col, h) for every register r whose element the fold reads
      // from accumulator dst_acc: D1's upper triangle i <= j and E columns, every D2 column.
      // A D1 entry's running fp64 sum lives in its owner thread's registers or shared slab slots (TcSums), or in L2:
      // there the add is a fire-and-forget reduction (red.add.f64, one IEEE fp64 add like `*p += v`).  Each element has
      // one writer, whose store and reductions to it take effect in program order (same-address coherence), so every
      // home holds the same sum: the chunks' values added in chunk order with round-to-nearest.  The on-chip homes keep
      // the drain off L2, where the ~9 300 reductions per CTA of a drain, issued by all SMs after the same number of
      // tiles, stalled every SM's stream of loads at once.
      using H = TcSums<DFIX, SPLIT, RAWB, EW, WG>;
      double* my_part = part + (size_t)blockIdx.x * kTcAccElems;
      double sums[H::kRegs > 0 ? H::kRegs : 1];
      // off: the development knob that sends every entry through L2
      const bool on_chip_off = (dbg & 256u) != 0u;
      auto slab_addr = [&](int s, int ln) {
        return sbase + G::kOffSlab + (uint32_t)(((4 * H::kSlabBase + (warp & 3) * H::kSlab + s) * 32 + ln) * 8);
      };
      auto store = [&](auto n_regs, int dst_acc, int col0, bool add, auto val) {
        // the lane is re-read here: partial indices computed from a kept one are hoisted out of the tile loop and hold a
        // register each
        const int ln = (int)lane_id(), row0 = 64 * WG + 16 * (warp & 3) + (ln >> 2);
#pragma unroll
        for (int r = 0; r < decltype(n_regs)::value; ++r) {
          const int col = col0 + 8 * (r >> 2) + 2 * (ln & 3) + (r & 1), h = (r >> 1) & 1, i = row0 + 8 * h;
          const bool lower = dst_acc == 0 && col < kTcM && i > col;   // D1's lower triangle: (col, i) holds it
          const double v = val(r, col, h);
          const bool on_chip = dst_acc == 0 && r >= H::kFirstSlab;
          if (on_chip && r >= H::kFirstReg) {
            double& s = sums[r - H::kFirstReg];
            s = add ? __dadd_rn(s, v) : v;
          } else if (on_chip) {
            const uint32_t a = slab_addr(r - H::kFirstSlab, ln);
            st_shared_f64_if(a, add ? __dadd_rn(ld_shared_f64(a), v) : v, !on_chip_off);
          }
          put_f64(my_part + tc_part_index(dst_acc, i, col, EW), v, add, !lower && (!on_chip || on_chip_off));
        }
      };
      // the end of the range: the on-chip sums to their partial entries
      auto flush = [&]() {
        const int ln = (int)lane_id(), row0 = 64 * WG + 16 * (warp & 3) + (ln >> 2);
#pragma unroll
        for (int r = H::kFirstSlab; r < H::kR1; ++r) {
          const int col = kC1 + 8 * (r >> 2) + 2 * (ln & 3) + (r & 1), i = row0 + 8 * ((r >> 1) & 1);
          const double s = r >= H::kFirstReg ? sums[r - H::kFirstReg] : ld_shared_f64(slab_addr(r - H::kFirstSlab, ln));
          put_f64(my_part + tc_part_index(0, i, col, EW), s, false, !(col < kTcM && i > col) && !on_chip_off);
        }
      };
      // RAWB's feature columns carry the raw x: sum_r a_i x_j - c_j sum_r a_i = sum_r a_i v_j, where sum_r a_i is E's ones
      // column (registers kF / 2 and kF / 2 + 2, held by lane 4 * (lane / 4))
      auto drain = [&](const auto& acc, int dst_acc, int col0, bool add) {
        constexpr int kR = sizeof(acc) / sizeof(float);
        if constexpr (RAWB) {
          constexpr int kF = 2 * kR - EW;
          const double s1[2] = {(double)__shfl_sync(0xffffffffu, acc[kF / 2], lane & ~3),
                                (double)__shfl_sync(0xffffffffu, acc[kF / 2 + 2], lane & ~3)};
          store(std::integral_constant<int, kR>{}, dst_acc, col0, add, [&](int r, int col, int h) {
            return col < kTcM ? (double)acc[r] - (double)shift_s[col] * s1[h] : (double)acc[r];
          });
        } else {
          store(std::integral_constant<int, kR>{}, dst_acc, col0, add, [&](int r, int, int) { return (double)acc[r]; });
        }
      };
      // the stages of a tile: RAWB's consumers also hold its raw stage, the B operand of its MMAs
      auto release = [&](int tile) {
        mbar_arrive(bar_op_empty + 8 * (tile % kOpStages));
        if constexpr (RAWB) mbar_arrive(bar_raw_empty + 8 * (tile % kRawStages));
      };
      constexpr uint32_t a_off = (uint32_t)WG * 8 * kOpSBO;      // this warpgroup's 64 features of A
      int os = 0, held = -1, in_chunk = 0;                       // held: the tile whose stages wait for their MMAs
      uint32_t oph = 0;
      bool first_chunk = true;
      for (int it = 0; it < my_tiles; ++it) {
        mbar_wait(bar_op_full + 8 * os, oph, wait_ns);
        const uint32_t op_addr = sbase + kOffOp + os * kOpStageBytes;
        wgmma_fence();
#pragma unroll
        for (int k2 = 0; k2 < kTcRows / 16; ++k2) {
          const uint32_t k_addr = op_addr + k2 * 2 * kOpLBO;
          const uint64_t hi_desc = make_smem_desc(k_addr + a_off), lo_desc = make_smem_desc(k_addr + kOpLoOff + a_off);
          const uint32_t sc1 = (in_chunk > 0 || k2 > 0) ? 1u : 0u, sc2 = (it > 0 || k2 > 0) ? 1u : 0u;
          if constexpr (RAWB) {
            // rows 16 k2 .. 16 k2 + 15 of the raw tile from box WG (features 64 WG on), and E
            const uint64_t x_desc = make_raw_desc(sbase + kOffRaw + (uint32_t)(it % kRawStages) * kRawStageBytes +
                                                  (uint32_t)WG * kRawBoxBytes + k2 * 16 * 128);
            const uint64_t e_desc = make_smem_desc(k_addr + kOpEOff);
            if (!(dbg & 2u)) {
              wgmma<kF1, 1>(acc1, hi_desc, x_desc, sc1);
              wgmma<EW, 0>(acc1 + kF1 / 2, hi_desc, e_desc, sc1);
            }
            if (SPLIT && !(dbg & 3u)) {
              wgmma<kF2, 1>(acc2, lo_desc, x_desc, sc2);
              wgmma<EW, 0>(acc2 + kF2 / 2, lo_desc, e_desc, sc2);
            }
          } else {
            if (!(dbg & 2u)) wgmma<kF1 + EW, 0>(acc1, hi_desc, make_smem_desc(k_addr + a_off), sc1);   // [hi_WG.. | E]
            if (SPLIT && !(dbg & 3u)) wgmma<kF2 + EW, 0>(acc2, lo_desc, make_smem_desc(k_addr), sc2);   // [hi | E]
          }
        }
        wgmma_commit();
        const bool last = (in_chunk == chunk_tiles - 1) || (it == my_tiles - 1);
        // the previous tile's MMAs are complete after wait_group 1 (this tile's too after wait_group 0): free their
        // stages; the last tile of the range is always `last`, so the accumulators are settled when the loop ends
        if (last) {
          wgmma_wait<0>();
          fence_regs(acc1);
          if constexpr (SPLIT) fence_regs(acc2);
        } else {
          wgmma_wait<1>();
        }
        if (lane == 0) {
          if (held >= 0) release(held);
          if (last) release(it);
        }
        held = last ? -1 : it;
        if (last) {
          drain(acc1, 0, kC1, !first_chunk);                     // D1 of this chunk
          first_chunk = false;
          in_chunk = 0;
        } else {
          ++in_chunk;
        }
        if (++os == kOpStages) { os = 0; oph ^= 1; }
      }
      wgmma_wait<0>();   // a no-op at run time (see above), but ptxas cannot prove it and would wait inside the loop
      // A = lo accumulated over the whole range (small zero-mean sums): D2, or with RAWB added into D1 after its last
      // drain (same thread, same element: program order)
      if constexpr (SPLIT) {
        fence_regs(acc2);
        drain(acc2, RAWB ? 0 : 1, RAWB ? kC1 : 0, RAWB);
      }
      flush();
    };
    // branch on a shuffled warp index: ptxas serialises the wgmma of both copies when the branch depends on the thread
    // index directly (it cannot tell that the condition is uniform over each warpgroup)
    if (__shfl_sync(0xffffffffu, warp, 0) >= 4) consume(std::integral_constant<int, 1>{});
    else consume(std::integral_constant<int, 0>{});
  } else {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(G::kProducerRegs));
    // ===== producers: eight transform warps, two on each SM sub-partition =====
    // Lane 0 of kTmaWarp also issues the TMA loads, G::kAhead tiles ahead of its own transform.  kEWarp also writes the
    // E columns [1, y'_hi, y'_lo] of the whole tile and sums y', y'^2, rows on CUDA cores: one warp, so that each
    // lane's fp32 sum over a tile covers the same rows in the same order for every split of the work.
    const uint32_t tx = (uint32_t)(kTcRows * d * sizeof(T)) + kTcRows * pack * 4 + (has_mask ? kTcRows * pack : 0);
    auto issue = [&](int j) {                   // TMA loads of tile j
      const int s = j % kRawStages;
      mbar_wait(bar_raw_empty + 8 * s, ((uint32_t)(j / kRawStages) & 1u) ^ 1u, wait_ns);
      const uint32_t full = bar_raw_full + 8 * s;
      mbar_expect_tx(full, tx);
      const int64_t row0 = (tile_begin + j) * kTcRows;
      tma_load_2d(sbase + kOffRaw + s * kRawStageBytes, &tmX, 0, (int)row0, full);
      if constexpr (RAWB) tma_load_2d(sbase + kOffRaw + s * kRawStageBytes + kRawBoxBytes, &tmX, 64, (int)row0, full);
      const int sub0 = (int)row0 * pack;                               // first original row of the tile
      if (y_map_2d) tma_load_2d(sbase + kOffY + s * kYStageBytes, &tmY, 0, sub0 >> 2, full);
      else tma_load_1d(sbase + kOffY + s * kYStageBytes, &tmY, sub0, full);
      if (has_mask == 2) tma_load_2d(sbase + kOffMask + s * kMStageBytes, &tmM, 0, sub0 >> 4, full);
      else if (has_mask) tma_load_1d(sbase + kOffMask + s * kMStageBytes, &tmM, sub0, full);
    };
    const bool issuer = warp == kTmaWarp && lane == 0;
    if (issuer)
      for (int j = 0; j < G::kAhead && j < my_tiles; ++j) issue(j);

    // Transform: shift, bf16 hi/lo split, K-major operand store.  A lane owns the adjacent features i, i + 1 of a
    // 64-feature block (one 8- or 4-byte load per row); a task is (block, 8-row K group g): nb * 8 tasks per tile.
    // nb (1 or 2) divides kXformWarps, so a warp always converts the same block and loads its shifts once per tile.
    const int t = warp - kFirstXformWarp;
    const int nb = (d + 63) >> 6;
    const int i = 64 * (t % nb) + 2 * lane;
    // Store order: the lanes of a quarter warp write 8 different 16-byte columns of the 128-byte core-matrix rows only
    // if half of them store feature i + 1 first (features i and i + 1 share a bank group otherwise).
    const uint32_t swp = ((uint32_t)lane >> 2) & 1u;
    const uint32_t st_off = (uint32_t)((i >> 3) * kOpSBO + (i & 7) * 16);
    // kEWarp's per-lane sums of y', y'^2, rows live in shared memory, and their address is recomputed where it is used:
    // registers are what the transform is short of
    auto esum = [&]() { return sbase + G::kOffESum + 8 * lane_id(); };
    if (warp == kEWarp) { st_shared_f64(esum(), 0.0); st_shared_f64(esum() + 256, 0.0); st_shared_f64(esum() + 512, 0.0); }
    int rs = 0, os = 0;
    uint32_t rph = 0, oph = 0;
    for (int it = 0; it < my_tiles; ++it) {
      if (issuer && it + G::kAhead < my_tiles) issue(it + G::kAhead);
      __syncwarp();      // reconverge kTmaWarp: its lanes must not run the transform below in two divergent passes
      mbar_wait(bar_raw_full + 8 * rs, rph, wait_ns);
      mbar_wait(bar_op_empty + 8 * os, oph ^ 1, wait_ns);
      const int64_t row0 = (tile_begin + it) * kTcRows;
      const int64_t left = n_rows - row0;
      const int rows_valid = left < kTcRows ? (int)left : kTcRows;
      const bool full_tile = (!has_mask) && (rows_valid == kTcRows);
      const uint32_t raw_addr = sbase + kOffRaw + rs * kRawStageBytes;
      const uint32_t m_addr = sbase + kOffMask + rs * kMStageBytes;
      const uint32_t op_addr = sbase + kOffOp + os * kOpStageBytes;
      if (warp == kEWarp && !(dbg & 192u)) {
        const uint32_t y_addr = sbase + kOffY + rs * kYStageBytes;
        const uint32_t e_addr = op_addr + kOpEOff;
        const float c_y = shift_s[kMaxD];
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
              const uint32_t row = raw_addr + (uint32_t)rr * 128;
              const uint32_t z[4] = {0u, 0u, 0u, 0u};
#pragma unroll
              for (int q = 0; q < 8; ++q) { st_shared_v4(row + 16 * q, z); st_shared_v4(row + kRawBoxBytes + 16 * q, z); }
            }
            a += yv;
            b = fmaf(yv, yv, b);
            c += use ? 1.f : 0.f;
          }
        }
        const uint32_t es = esum();
        st_shared_f64(es, ld_shared_f64(es) + (double)a);
        st_shared_f64(es + 256, ld_shared_f64(es + 256) + (double)b);
        st_shared_f64(es + 512, ld_shared_f64(es + 512) + (double)c);
      }
      if (i < d && !(dbg & 128u)) {
        float c_i[2];                               // (a volatile load: kept out of the registers live across tiles)
        ld_vals_vec<float, 2>(sbase + G::kOffShift + 4 * (uint32_t)i, c_i);
        for (int g = t / nb; g < kKGroups; g += kXformWarps / nb) {
          const int r0 = g * 8;
          float v0[8], v1[8];                       // features i, i + 1 of rows r0 .. r0 + 7
          const uint32_t src = raw_addr + (uint32_t)r0 * ((uint32_t)d * sizeof(T)) + (uint32_t)i * sizeof(T);
#pragma unroll
          for (int k = 0; k < 8; ++k) {
            // RAWB: feature i of row r0 + k sits in box i / 64, 16-byte chunk ((i % 64) / 8) ^ k of the 128-byte row
            const uint32_t a = RAWB ? raw_addr + (uint32_t)(i >> 6) * kRawBoxBytes + (uint32_t)(r0 + k) * 128 +
                                          ((((uint32_t)(i & 63) >> 3) ^ (uint32_t)k) << 4) + (uint32_t)(i & 7) * 2
                                    : src + (uint32_t)k * ((uint32_t)d * sizeof(T));
            float x[2];
            if (dbg & 8u) { x[0] = __uint_as_float(src + k); x[1] = __uint_as_float(src - k); }
            else ld_vals_vec<T, 2>(a, x);
            v0[k] = x[0] - c_i[0];
            v1[k] = x[1] - c_i[1];
          }
          if (!full_tile) {
            const int blk = i / d_orig;             // which original row of the super-row features i, i + 1 belong to
#pragma unroll
            for (int k = 0; k < 8; ++k) {
              bool use = (r0 + k) < rows_valid;
              if (use && has_mask) use = (ld_shared_u8(m_addr + (r0 + k) * pack + blk) == (uint32_t)keep);
              if (!use) { v0[k] = 0.f; v1[k] = 0.f; }
            }
          }
          uint32_t h0[4], l0[4], h1[4], l1[4];
#pragma unroll
          for (int p = 0; p < 4; ++p) {
            if constexpr (SPLIT) {
              split2(v0[2 * p], v0[2 * p + 1], h0[p], l0[p]);
              split2(v1[2 * p], v1[2 * p + 1], h1[p], l1[p]);
            } else {
              const __nv_bfloat162 e0 = __floats2bfloat162_rn(v0[2 * p], v0[2 * p + 1]);
              const __nv_bfloat162 e1 = __floats2bfloat162_rn(v1[2 * p], v1[2 * p + 1]);
              h0[p] = *reinterpret_cast<const uint32_t*>(&e0);
              h1[p] = *reinterpret_cast<const uint32_t*>(&e1);
              l0[p] = l1[p] = 0u;
            }
          }
          if (!(dbg & 4u)) {
            const uint32_t dst = op_addr + (uint32_t)g * kOpLBO + st_off;
            uint32_t f[4], s[4];                    // first / second store: feature i + swp, then i + 1 - swp
#pragma unroll
            for (int p = 0; p < 4; ++p) { f[p] = swp ? h1[p] : h0[p]; s[p] = swp ? h0[p] : h1[p]; }
            st_shared_v4(dst + 16 * swp, f);
            st_shared_v4(dst + 16 - 16 * swp, s);
            if constexpr (SPLIT) {
#pragma unroll
              for (int p = 0; p < 4; ++p) { f[p] = swp ? l1[p] : l0[p]; s[p] = swp ? l0[p] : l1[p]; }
              st_shared_v4(dst + kOpLoOff + 16 * swp, f);
              st_shared_v4(dst + kOpLoOff + 16 - 16 * swp, s);
            }
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
    if (warp == kEWarp) {
      const uint32_t es = esum();
      double sy = ld_shared_f64(es), syy = ld_shared_f64(es + 256), cnt = ld_shared_f64(es + 512);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        sy += __shfl_xor_sync(0xffffffffu, sy, o);
        syy += __shfl_xor_sync(0xffffffffu, syy, o);
        cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
      }
      if (lane == 0) {
        double* ys = part + (size_t)gridDim.x * kTcAccElems + kTcSums * blockIdx.x;   // behind all accumulators
        ys[0] = sy; ys[1] = syy; ys[2] = cnt;
      }
    }
  }
}

// What tc_finalize_kernel does after the reduce + fold (passed by value).
struct TcFinal {
  int assign;                 // S = value instead of S += value (first writer of a fresh statistic)
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
constexpr int kFinalizeCtas = (kRedElems + kFinalizeThreads / 4 - 1) / (kFinalizeThreads / 4);   // 113: one pass

__global__ void __launch_bounds__(kFinalizeThreads, 1)
tc_finalize_kernel(const double* part, int n_ctas, double* red, const float* __restrict__ shift, int d, int pack,
                   int ew, int d2, double* S, unsigned int* sync, const TcFinal fin) {
  __shared__ double quarter[kFinalizeThreads];
  __shared__ double c_s[kMaxD + 1];                              // the shift as fp64 (c_s[kMaxD]: c_y)
  for (int j = threadIdx.x; j <= kMaxD; j += blockDim.x) c_s[j] = (double)shift[j];
  {
    constexpr int epb = kFinalizeThreads / 4;                    // elements per pass of a CTA
    const int n_acc = tc_part_elems(ew, d2 != 0);                // the entries the Gram launch wrote
    const int n_red = n_acc + kTcSums;
    const int per = (((n_red + (int)gridDim.x - 1) / (int)gridDim.x) + epb - 1) / epb * epb;
    const int e0 = (int)blockIdx.x * per;
    const int e1 = e0 + per < n_red ? e0 + per : n_red;
    if (e0 < n_red) tc_reduce_range(part, n_ctas, n_acc, red, e0, e1, quarter);
  }
  grid_barrier(sync + 0);
  {
    const int dp = d + 2;
    const int total = dp * dp;
    const size_t slot = xchg_slot_offset(fin.epoch, fin.rank);
    for (int idx = (int)(blockIdx.x * blockDim.x + threadIdx.x); idx < total; idx += (int)(gridDim.x * blockDim.x)) {
      const double val = tc_fold_value(red, c_s, d, pack, ew, d2 != 0, idx);
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

bool gram_tc_supported(const void* X, int x_dtype, const float* y, int64_t n, int d, int64_t ldx,
                       const uint8_t* mask) {
  const int es = x_dtype == B2_F32 ? 4 : 2;
  if (d < 4 || d > kMaxD) return false;
  if ((d * es) % 16 != 0) return false;
  if ((ldx * es) % 16 != 0) return false;
  if ((reinterpret_cast<uintptr_t>(X) & 15) != 0 || (reinterpret_cast<uintptr_t>(y) & 15) != 0) return false;
  if (mask != nullptr && (reinterpret_cast<uintptr_t>(mask) & 15) != 0) return false;
  if (n < kTcRows) return false;
  if (n > (int64_t)0x7fffffff) return false;  // TMA coordinates are int32
  return true;
}

// A vector of n elements of es bytes (y, the row mask) read `box` elements per tile: a 1-D map, else a [n / k][k] view
// with 16-byte rows (k = 16 / es) that lands the same bytes in shared memory.  Box extents stop at 256 (pack = 5 tiles
// read 320), and a driver may refuse rank-1 maps.  The view is taken only when k divides n: otherwise its last row
// would reach past the vector.
static int encode_vec(PFN_encodeTiled encode, CUtensorMap* tm, CUtensorMapDataType type, int es, const void* v,
                      int64_t n, cuuint32_t box, int* view_2d, const char* what) {
  const cuuint32_t estr[2] = {1, 1};
  const cuuint64_t dims[1] = {(cuuint64_t)n}, strides[1] = {0};
  CUresult r = CUDA_ERROR_INVALID_VALUE;
  if (box <= 256)
    r = encode(tm, type, 1, const_cast<void*>(v), dims, strides, &box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  *view_2d = r != CUDA_SUCCESS;
  const int k = 16 / es;
  if (r != CUDA_SUCCESS && n % k == 0) {
    const cuuint64_t dims2[2] = {(cuuint64_t)k, (cuuint64_t)(n / k)}, strides2[1] = {16};
    const cuuint32_t box2[2] = {(cuuint32_t)k, box / k};
    r = encode(tm, type, 2, const_cast<void*>(v), dims2, strides2, box2, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  }
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(%s) failed with %d (n=%lld box=%u)", what, (int)r, (long long)n, (unsigned)box);
    return B2_E_CUDA;
  }
  return B2_OK;
}

// d: inner extent of the (super-)row tensor; d_box: inner extent of the smem tile (> d: the rest is zero fill)
// swz64: the raw tile of the bf16 D = 128 path -- [64 rows][64 features] boxes (128-byte rows) with SWIZZLE_128B
static int encode_maps(PFN_encodeTiled encode, const void* X, int x_dtype, int es, const float* y, int64_t n, int d,
                       int d_box, int64_t ldx, int64_t n_y, int pack, const uint8_t* mask, bool swz64, CUtensorMap* tmX_out,
                       CUtensorMap* tmY_out, CUtensorMap* tmM_out, int* y_map_2d_out, int* m_map_2d_out) {
  const cuuint32_t y_box = (cuuint32_t)(kTcRows * pack);   // original rows per tile
  CUtensorMap& tmX = *tmX_out;
  memset(tmM_out, 0, sizeof(*tmM_out));
  *m_map_2d_out = 0;
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
  if (int r = encode_vec(encode, tmY_out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, y, n_y, y_box, y_map_2d_out, "y")) return r;
  if (mask == nullptr) return B2_OK;
  return encode_vec(encode, tmM_out, CU_TENSOR_MAP_DATA_TYPE_UINT8, 1, mask, n_y, y_box, m_map_2d_out, "mask");
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
                   const uint8_t* mask, int keep, bool assign, unsigned int scatter_epoch) {
  PFN_encodeTiled encode = get_encode();
  if (encode == nullptr) {
    set_error("cuTensorMapEncodeTiled is not available from the driver");
    return B2_E_CUDA;
  }
  const int es = x_dtype == B2_F32 ? 4 : 2;
  // Row packing: `pack` contiguous rows of 17..64 features are viewed as one super-row of pack * d_in <= 128 columns
  // ([n / pack][pack * d_in], zero-filled by TMA to the 128-wide tile) and run on the D = 128 fast path; the diagonal
  // d_in x d_in blocks of the 128 x 128 Gram sum to the true statistic (tc_fold_value).  The tensor maps cover a
  // multiple of lcm(pack, 16) rows (the y / mask views are 16-byte rows); the caller runs the < 80 leftover rows on
  // the CUDA-core kernel.
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
  b2_ctx::TmCache& tc = ctx->tm_cache;
  const bool cached = tc.X == X && tc.y == y && tc.mask == mask && tc.n == n_in && tc.ldx == ldx_in && tc.d == d_in &&
                      tc.x_dtype == x_dtype;
  if (cached) {
    memcpy(&tmX, tc.tmX, sizeof(tmX)); memcpy(&tmY, tc.tmY, sizeof(tmY)); memcpy(&tmM, tc.tmM, sizeof(tmM));
  } else {
    int y_map_2d = 0, m_map_2d = 0;
    if (int r = encode_maps(encode, X, x_dtype, es, y, n, d_tensor, d, ldx, n_y, pack, mask, rawb, &tmX, &tmY, &tmM, &y_map_2d,
                            &m_map_2d))
      return r;
    tc.X = X; tc.y = y; tc.mask = mask; tc.n = n_in; tc.ldx = ldx_in; tc.d = d_in; tc.x_dtype = x_dtype;
    tc.y_map_2d = y_map_2d; tc.m_map_2d = m_map_2d;
    memcpy(tc.tmX, &tmX, sizeof(tmX)); memcpy(tc.tmY, &tmY, sizeof(tmY)); memcpy(tc.tmM, &tmM, sizeof(tmM));
  }

  const int64_t total_tiles = (n + kTcRows - 1) / kTcRows;
  const int sms = (ctx->sm_limit > 0 && ctx->sm_limit < ctx->sm_count) ? ctx->sm_limit : ctx->sm_count;
  const int grid = (int)(total_tiles < sms ? total_tiles : sms);
  // the RAWB accumulators carry the unshifted x (sum hi_i x_j includes c_j sum hi_i): a quarter of the fp32 chain length
  // keeps their truncation error at the level of the shifted operands' accumulators
  int chunk_tiles = ctx->drain_rows / kTcRows / (rawb ? 4 : 1);
  if (chunk_tiles < 1) chunk_tiles = 1;

#ifdef B2_DEV_KNOBS
  static const uint32_t wait_ns = []() {   // development knob: suspend-time hint of the pipeline waits
    const char* e = getenv("B2_WAIT_HINT_NS");
    return e ? (uint32_t)atoi(e) : 20000u;
  }();
#else
  constexpr uint32_t wait_ns = 20000u;     // try_wait suspend hint (ns); measured insensitive 0..20000 (r01)
#endif
#ifdef B2_DEV_KNOBS
  static const uint32_t dbg = []() {       // ablations: bit0 skip MMA2, bit1 skip all MMAs, bit2 skip STS, bit3 skip LDS, bit5 skip proxy fence,
                                           // bit6 skip the E columns and the y' sums, bit7 skip the whole transform
    const char* e = getenv("B2_TC_DEBUG");
    return e ? (uint32_t)atoi(e) : 0u;
  }();                                     // bit8 every drained D1 sum in L2 (no on-chip homes; results unchanged)
#else
  constexpr uint32_t dbg = 0u;
#endif
  // the E columns the MMAs cover, and whether the launch writes D2 (hi + lo operands without RAWB): the finalize reads
  // exactly the partial entries these two select
  const bool split = ctx->precision == B2_PRECISION_SPLIT;
  const int ew = tc_e_width(pack);
  const bool d2 = split && !rawb;
  decltype(&gram_tc_kernel<float, 0, false>) kernel = nullptr;
  uint32_t smem = TcGeo<false>::kSmemBytes;
  with_rows(x_dtype, X, [&](auto* Xr) {
    using T = row_t<decltype(Xr)>;
    return with_int<0, 1>(split, [&](auto SP) {
      constexpr bool kSplit = decltype(SP)::value;
      if (d != 128) kernel = gram_tc_kernel<T, 0, kSplit>;                   // runtime d: never packed (ew = 8)
      else if (ew == 16) kernel = gram_tc_kernel<T, 128, kSplit, false, 16>;
      else kernel = gram_tc_kernel<T, 128, kSplit>;
      if constexpr (std::is_same_v<T, __nv_bfloat16>) {
        if (rawb) {
          kernel = gram_tc_kernel<T, 128, kSplit, true>;
          smem = TcGeo<true>::kSmemBytes;
        }
      }
      return B2_OK;
    });
  });
  // set before the start event: the call's host latency is not part of the kernel time the events report
  B2_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  const int pair = ctx->k_pairs % kKernelEventPairs;
  B2_CUDA(cudaEventRecord(ctx->ev_k[pair][0], ctx->stream));
  kernel<<<grid, kThreads, smem, ctx->stream>>>(tmX, tmY, tmM, tc.y_map_2d, mask != nullptr ? 1 + tc.m_map_2d : 0, keep,
                                                n, d, pack, d_in, ctx->shift, chunk_tiles, ctx->tc_part, wait_ns, dbg);
  B2_CUDA(cudaGetLastError());
  B2_CUDA(cudaEventRecord(ctx->ev_k[pair][1], ctx->stream));
  ctx->k_pairs += 1;

  // finalize: reduce + fold (+ peer scatter) in one cooperative launch
  TcFinal fin;
  memset(&fin, 0, sizeof(fin));
  fin.assign = assign ? 1 : 0;
  fin.n_ranks = 1;
  if (scatter_epoch != 0) {
    fin.n_ranks = ctx->n_ranks; fin.rank = ctx->rank; fin.epoch = scatter_epoch;
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
    const double* part_arg = ctx->tc_part;
    const float* shift_arg = ctx->shift;
    B2_CUDA(cudaLaunchKernelEx(&cfg, tc_finalize_kernel, part_arg, grid, ctx->tc_red, shift_arg, d_in, pack, ew,
                               d2 ? 1 : 0, ctx->S, ctx->tc_sync, fin));
  }
  ctx->launches += 2;
  return B2_OK;
}

}  // namespace b2
