// score.cu -- batch scoring yhat = X.coef + intercept fused with the hold-out metric reductions.
//
// Replaces  ols_regressor.predict(X_test)        stage_1_train_model.py:107
//           model.predict(X)                     stage_2_serve_model.py:78
//           model_metrics(y_actual, y_predicted) stage_1_train_model.py:79-90
//             MAPE = mean(|yhat-y| / max(|y|, eps_f64)), R^2 = 1 - SSres/SStot, max_error = max|y-yhat|
//
// HBM-bound: one pass over X (D*sizeof(x) bytes per row) + 4 B (y) + 4 B (yhat).  One warp per
// row, 128-bit loads, the dot product and all reductions in fp64 (products of an fp32 value with
// an fp64 coefficient; this reproduces the float64 predict of the oracle to ~1e-13).
#include <cuda_bf16.h>

#include "b2_internal.cuh"
#include "b2_ptx.cuh"

namespace b2 {
namespace {

constexpr int kScoreThreads = 256;
constexpr int kScoreWarps = kScoreThreads / 32;
constexpr double kEpsF64 = 2.220446049250313e-16;

// The per-row statistics are the fp64-pipe cost of scoring (they bind the narrow-row and bf16 kernels), so they are kept
// to 13 fp64 instructions: one residual, one reciprocal refined by a single Newton step from the fp32 seed (the seed is
// good to 2^-23, one step gives 2^-46 = 1.4e-14 relative -- the parity bar is 1e-12), fused multiply-adds for the four
// second moments, the range test on the fp32 copy of |y|, and an integer row counter.
struct RowStats {
  double ape = 0.0, sse = 0.0, sy = 0.0, syy = 0.0, mx = 0.0, sp = 0.0, spp = 0.0, syp = 0.0, mxape = 0.0;
  int rows = 0;
  __device__ __forceinline__ double cnt() const { return (double)rows; }
  __device__ __forceinline__ void add(double y, double p) {
    const double r = y - p;
    const double e = fabs(r);
    const double ay = fabs(y);
    const float ayf = (float)ay;
    // |y| in the float range (the overwhelmingly common case): one cheap reciprocal serves both APE terms
    const bool common = ayf > 1e-30f && ayf < 1e30f;
    double term, rel;
    if (common) {
      double rc = (double)__frcp_rn(ayf);
      rc = fma(rc, fma(-ay, rc, 1.0), rc);
      term = e * rc;
      rel = term;
    } else {
      term = e / fmax(ay, kEpsF64);               // sklearn MAPE clamp (stage_1_train_model.py:81)
      rel = e / ay;                               // |score/label - 1| (stage_4...:89,104); inf when label == 0
    }
    ape += term;
    sse = fma(r, r, sse);
    sy += y;
    syy = fma(y, y, syy);
    mx = fmax(mx, e);
    rows += 1;
    sp += p;                                      // Pearson correlation terms (stage_4...:103 "r_squared")
    spp = fma(p, p, spp);
    syp = fma(y, p, syp);
    mxape = fmax(mxape, rel);
  }
  // Branch-free flavour for rows whose |y| is in the float range (checked per warp by the caller): the row is dropped
  // by zeroing its inputs (use == false), so several rows per lane interleave without control flow between them.
  // y arrives as the fp32 value it was stored as: the range test and the reciprocal seed need no fp64 conversion.
  __device__ __forceinline__ void add_fast(float yf, double p, bool use) {
    const double y = (double)(use ? yf : 0.f);
    const double ps = use ? p : 0.0;
    float rcf;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(rcf) : "f"(use ? fabsf(yf) : 1.f));
    const double r = y - ps;
    const double e = fabs(r);
    double rc = (double)rcf;
    rc = fma(rc, fma(-fabs(y), rc, 1.0), rc);     // one Newton step: 2^-23 -> 2^-46 (use == false: finite, e == 0)
    const double term = e * rc;
    ape += term;
    sse = fma(r, r, sse);
    sy += y;
    syy = fma(y, y, syy);
    mx = fmax(mx, e);
    rows += use ? 1 : 0;
    sp += ps;
    spp = fma(ps, ps, spp);
    syp = fma(y, ps, syp);
    mxape = fmax(mxape, term);
  }
  // same ten statistics with correctly rounded divisions (b2_metrics: parity with the float64 reference to rounding)
  __device__ __forceinline__ void add_exact(double y, double p) {
    const double r = y - p, e = fabs(r), ay = fabs(y);
    ape += e / fmax(ay, kEpsF64);
    sse = fma(r, r, sse);
    sy += y; syy = fma(y, y, syy);
    mx = fmax(mx, e);
    rows += 1;
    sp += p; spp = fma(p, p, spp); syp = fma(y, p, syp);
    mxape = fmax(mxape, e / ay);
  }
  // in the stats_out order of include/b2gram.h
  __device__ __forceinline__ void values(double (&v)[kNStats]) const {
    v[0] = ape; v[1] = sse; v[2] = sy; v[3] = syy; v[4] = mx; v[5] = cnt(); v[6] = sp; v[7] = spp; v[8] = syp; v[9] = mxape;
  }
};
__device__ __forceinline__ bool stat_is_max(int k) { return k == 4 || k == 9; }
__device__ __forceinline__ double shfl_xor_d(double v, int m) { return __shfl_xor_sync(0xffffffffu, v, m); }

// ---- the CTA reductions: statistics combined across lanes 16, 8, ..., LAST of a warp, then one warp's values in
// red[warp] (lane 0 stores), then the NW warps in order into part[blockIdx.x]; the gradient sums likewise ---------------
template <int LAST>
__device__ __forceinline__ void stats_butterfly(double (&v)[kNStats]) {
#pragma unroll
  for (int k = 0; k < kNStats; ++k) {
#pragma unroll
    for (int o = 16; o >= LAST; o >>= 1) {
      const double other = shfl_xor_d(v[k], o);
      v[k] = stat_is_max(k) ? fmax(v[k], other) : v[k] + other;
    }
  }
}
__device__ __forceinline__ void stats_store(double (*red)[kNStats], int warp, int lane, const double (&v)[kNStats]) {
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < kNStats; ++k) red[warp][k] = v[k];
  }
}
template <int NW>
__device__ __forceinline__ void stats_fold(const double (*red)[kNStats], double* __restrict__ part) {
  __syncthreads();
  if (threadIdx.x < kNStats) {
    const int k = threadIdx.x;
    double acc = 0.0;
    for (int w = 0; w < NW; ++w) acc = stat_is_max(k) ? fmax(acc, red[w][k]) : acc + red[w][k];
    part[(size_t)blockIdx.x * kNStats + k] = acc;
  }
}
// red[w] holds warp w's gradient sums at the features < d, at kMaxD (g_1) and at kMaxD + 1 (sum e^2); every other entry
// of the partial is zero
template <int NW>
__device__ __forceinline__ void grad_fold(const double (*red)[kGradOut], int d, double* __restrict__ part) {
  __syncthreads();
  for (int t = threadIdx.x; t < kGradOut; t += blockDim.x) {
    double v = 0.0;
    if (t < d || t >= kMaxD)
      for (int w = 0; w < NW; ++w) v += red[w][t];
    part[(size_t)blockIdx.x * kGradOut + t] = v;
  }
}

template <typename T>
__device__ __forceinline__ double lane_dot(const T* __restrict__ row, int d, int lane, const double* cf, bool vec);

template <>
__device__ __forceinline__ double lane_dot<float>(const float* __restrict__ row, int d, int lane, const double* cf,
                                                  bool vec) {
  double acc = 0.0;
  if (vec) {
    if (lane * 4 < d) {
      const float4 x = __ldg(reinterpret_cast<const float4*>(row) + lane);
      acc = fma((double)x.x, cf[0], acc);
      acc = fma((double)x.y, cf[1], acc);
      acc = fma((double)x.z, cf[2], acc);
      acc = fma((double)x.w, cf[3], acc);
    }
  } else {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int j = lane + 32 * k;
      if (j < d) acc = fma((double)__ldg(row + j), cf[k], acc);
    }
  }
  return acc;
}

template <>
__device__ __forceinline__ double lane_dot<__nv_bfloat16>(const __nv_bfloat16* __restrict__ row, int d, int lane,
                                                          const double* cf, bool vec) {
  double acc = 0.0;
  if (vec) {
    if (lane * 4 < d) {
      const uint2 u = __ldg(reinterpret_cast<const uint2*>(row) + lane);
      acc = fma((double)__uint_as_float(u.x << 16), cf[0], acc);
      acc = fma((double)__uint_as_float(u.x & 0xffff0000u), cf[1], acc);
      acc = fma((double)__uint_as_float(u.y << 16), cf[2], acc);
      acc = fma((double)__uint_as_float(u.y & 0xffff0000u), cf[3], acc);
    }
  } else {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int j = lane + 32 * k;
      if (j < d) acc = fma((double)__bfloat162float(row[j]), cf[k], acc);
    }
  }
  return acc;
}

template <typename T>
__global__ void __launch_bounds__(kScoreThreads)
score_kernel(const T* __restrict__ X, int64_t n, int d, int64_t ldx, const double* __restrict__ coef,
             const float* __restrict__ y, const uint8_t* __restrict__ mask, int keep, float* __restrict__ yhat,
             int vec, double* __restrict__ part) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double cf[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int j = vec ? lane * 4 + k : lane + 32 * k;
    cf[k] = j < d ? coef[j] : 0.0;
  }
  const double b0 = coef[kMaxD];
  RowStats st;
  const int64_t warps_total = (int64_t)gridDim.x * kScoreWarps;
  const int64_t gw = (int64_t)blockIdx.x * kScoreWarps + warp;
  constexpr int kU = 4;  // rows in flight per warp
  for (int64_t base = gw * kU; base < n; base += warps_total * kU) {
    double acc[kU];
    bool use[kU];
#pragma unroll
    for (int u = 0; u < kU; ++u) {
      const int64_t row = base + u;
      use[u] = row < n;
      if (use[u] && mask != nullptr) use[u] = (__ldg(mask + row) == (uint8_t)keep);
      acc[u] = use[u] ? lane_dot<T>(X + row * ldx, d, lane, cf, vec != 0) : 0.0;
    }
#pragma unroll
    for (int u = 0; u < kU; ++u) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc[u] += __shfl_xor_sync(0xffffffffu, acc[u], o);
    }
    if (lane == 0) {
#pragma unroll
      for (int u = 0; u < kU; ++u) {
        const int64_t row = base + u;
        if (row < n) {
          const double p = acc[u] + b0;
          if (yhat != nullptr) yhat[row] = use[u] ? (float)p : 0.f;
          if (use[u] && y != nullptr) st.add((double)__ldg(y + row), p);
        }
      }
    }
  }
  __shared__ double red[kScoreWarps][kNStats];
  double v[kNStats];
  st.values(v);
  stats_store(red, warp, lane, v);
  stats_fold<kScoreWarps>(red, part);
}

// ---- fast path (d % 4 == 0, 16-byte aligned rows): 4 rows per warp iteration, 32 warps per SM ---------------
// Each lane loads 16 B of each of 4 rows (independent 128-bit loads in flight), forms its 4-term partial dot in
// fp64, and the 4 x 32 partials are reduced with a transposing butterfly (6 double shuffles instead of 20): after
// it, lane l holds the full dot of row ((l >> 4) & 1) * 2 + ((l >> 3) & 1).  The 4 lanes with (l & 7) == 0 then
// update the statistics of their own row in parallel.
template <typename T>
__device__ __forceinline__ void load_row4(const T* __restrict__ row, int lane, bool pred, float (&x)[4]);
// Predicated streaming loads as volatile PTX: the compiler keeps the four row loads of an iteration in
// distinct registers and issues them back to back (with plain __ldg it re-used one register quad and
// serialised the loads -- ncu r01: every row's first conversion stalled on long_scoreboard).
template <>
__device__ __forceinline__ void load_row4<float>(const float* __restrict__ row, int lane, bool pred, float (&x)[4]) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %5, 0;\n\t"
      "mov.f32 %0, 0f00000000;\n\tmov.f32 %1, 0f00000000;\n\tmov.f32 %2, 0f00000000;\n\tmov.f32 %3, 0f00000000;\n\t"
      "@p ld.global.nc.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];\n\t}"
      : "=f"(x[0]), "=f"(x[1]), "=f"(x[2]), "=f"(x[3])
      : "l"(reinterpret_cast<const float4*>(row) + lane), "r"((int)pred));
}
template <>
__device__ __forceinline__ void load_row4<__nv_bfloat16>(const __nv_bfloat16* __restrict__ row, int lane, bool pred,
                                                         float (&x)[4]) {
  uint32_t u0, u1;
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %3, 0;\n\t"
      "mov.b32 %0, 0;\n\tmov.b32 %1, 0;\n\t"
      "@p ld.global.nc.L1::no_allocate.v2.b32 {%0, %1}, [%2];\n\t}"
      : "=r"(u0), "=r"(u1)
      : "l"(reinterpret_cast<const uint2*>(row) + lane), "r"((int)pred));
  x[0] = __uint_as_float(u0 << 16); x[1] = __uint_as_float(u0 & 0xffff0000u);
  x[2] = __uint_as_float(u1 << 16); x[3] = __uint_as_float(u1 & 0xffff0000u);
}

constexpr int kRowsPerIter = 4;

template <typename T>
__global__ void __launch_bounds__(kScoreThreads, 4)
score_kernel_rows8(const T* __restrict__ X, int64_t n, int d, int64_t ldx, const double* __restrict__ coef,
                   const float* __restrict__ y, const uint8_t* __restrict__ mask, int keep,
                   float* __restrict__ yhat, double* __restrict__ part) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool col_ok = lane * 4 < d;
  double cf[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) cf[k] = (lane * 4 + k < d) ? coef[lane * 4 + k] : 0.0;
  const double b0 = coef[kMaxD];
  const int my_row = ((lane >> 4) & 1) * 2 + ((lane >> 3) & 1);   // row (of 4) this lane owns after the reduce
  RowStats st;
  const int64_t warps_total = (int64_t)gridDim.x * kScoreWarps;
  const int64_t gw = (int64_t)blockIdx.x * kScoreWarps + warp;
  for (int64_t base = gw * kRowsPerIter; base < n; base += warps_total * kRowsPerIter) {
    float x[kRowsPerIter][4];
    unsigned use_bits = 0;
    float y_mine = 0.f;                           // this lane's row label, fetched together with the X loads
    if (y != nullptr && (lane & 7) == 0 && base + my_row < n) y_mine = __ldg(y + base + my_row);
#pragma unroll
    for (int r = 0; r < kRowsPerIter; ++r) {     // 4 independent 128-bit loads in flight per lane
      const int64_t row = base + r;
      bool use = row < n;
      if (use && mask != nullptr) use = (__ldg(mask + row) == (uint8_t)keep);
      use_bits |= (use ? 1u : 0u) << r;
      load_row4<T>(X + row * ldx, lane, use && col_ok, x[r]);
    }
    double p[kRowsPerIter];
#pragma unroll
    for (int r = 0; r < kRowsPerIter; ++r) {
      double a = (double)x[r][0] * cf[0];
      a = fma((double)x[r][1], cf[1], a);
      a = fma((double)x[r][2], cf[2], a);
      p[r] = fma((double)x[r][3], cf[3], a);
    }
    // transposing butterfly: keep the half of the rows selected by the lane bit, add the partner's copy
    double q2[2], q1;
    {
      const bool hi = (lane & 16) != 0;
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const double send = hi ? p[r] : p[r + 2];
        const double keepv = hi ? p[r + 2] : p[r];
        q2[r] = keepv + shfl_xor_d(send, 16);
      }
    }
    {
      const bool hi = (lane & 8) != 0;
      const double send = hi ? q2[0] : q2[1];
      const double keepv = hi ? q2[1] : q2[0];
      q1 = keepv + shfl_xor_d(send, 8);
    }
    q1 += shfl_xor_d(q1, 4);
    q1 += shfl_xor_d(q1, 2);
    q1 += shfl_xor_d(q1, 1);
    if ((lane & 7) == 0) {
      const int64_t row = base + my_row;
      if (row < n) {
        const bool use = (use_bits >> my_row) & 1u;
        const double pr = q1 + b0;
        if (yhat != nullptr) yhat[row] = use ? (float)pr : 0.f;
        if (use && y != nullptr) st.add((double)y_mine, pr);
      }
    }
  }
  // block reduce: first across the 4 row-owning lanes of each warp (lanes 0, 8, 16, 24), then across warps
  double v[kNStats];
  st.values(v);
  stats_butterfly<8>(v);
  __shared__ double red[kScoreWarps][kNStats];
  stats_store(red, warp, lane, v);
  stats_fold<kScoreWarps>(red, part);
}

// ---- streaming path (wide contiguous rows): TMA bulk copies -> smem ring -> the same 4-rows-per-warp arithmetic -------
// The register-fed kernel above tops out at ~0.67 of the HBM roofline: 32 warps x 4 x 16 B per lane = 64 KB in flight
// per SM is not enough at the loaded DRAM latency (ncu r01).  Here one producer lane keeps kTmStages x 32 KB of bulk
// copies in flight per SM (cp.async.bulk, mbarrier full/empty) and 16 consumer warps read their rows from shared
// memory, 8 lanes per row (a 3-step xor reduce, no selects) with the per-row statistics batched 32 rows at a time.
constexpr int kTmStages = 6;
constexpr int kTmWarps = 15;                       // consumer warps; warp kTmWarps is the producer (16 warps: 128 registers)
constexpr int kTmThreads = 32 * (kTmWarps + 1);
constexpr int kTmTileRowsMax = 240;                // rows per stage (y tile: 960 B)
constexpr uint32_t kTmXStage = 32768;
constexpr int kTmMaxSweeps = 4;
constexpr uint32_t kTmYStage = kTmTileRowsMax * 4;                // 960 (a multiple of 16: bulk-copy granularity)
constexpr uint32_t kTmOffY = kTmStages * kTmXStage;
constexpr uint32_t kTmOffBar = kTmOffY + kTmStages * kTmYStage;
constexpr uint32_t kTmSmem = kTmOffBar + 2 * kTmStages * 8 + 128;

template <typename T>
__device__ __forceinline__ void lds_row4(uint32_t addr, bool pred, float (&x)[4]);
template <>
__device__ __forceinline__ void lds_row4<float>(uint32_t addr, bool pred, float (&x)[4]) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %5, 0;\n\t"
      "mov.f32 %0, 0f00000000;\n\tmov.f32 %1, 0f00000000;\n\tmov.f32 %2, 0f00000000;\n\tmov.f32 %3, 0f00000000;\n\t"
      "@p ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];\n\t}"
      : "=f"(x[0]), "=f"(x[1]), "=f"(x[2]), "=f"(x[3])
      : "r"(addr), "r"((int)pred));
}
template <>
__device__ __forceinline__ void lds_row4<__nv_bfloat16>(uint32_t addr, bool pred, float (&x)[4]) {
  uint32_t u0, u1;
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %3, 0;\n\t"
      "mov.b32 %0, 0;\n\tmov.b32 %1, 0;\n\t"
      "@p ld.shared.v2.b32 {%0, %1}, [%2];\n\t}"
      : "=r"(u0), "=r"(u1)
      : "r"(addr), "r"((int)pred));
  x[0] = __uint_as_float(u0 << 16); x[1] = __uint_as_float(u0 & 0xffff0000u);
  x[2] = __uint_as_float(u1 << 16); x[3] = __uint_as_float(u1 & 0xffff0000u);
}

// rows [0, n_tiles * tile_rows) of a contiguous matrix (ldx == d).  LPR lanes share a row (8: up to 128 features,
// 4: up to 64, 2: up to 32), 32 / LPR rows per warp iteration, tile_rows = sweeps * 15 * 32 / LPR.  The row mask
// (1 byte per row) is read straight from global memory, prefetched before the wait on the tile's barrier.
template <typename T, int LPR>
__global__ void __launch_bounds__(kTmThreads, 1)
score_tma_kernel(const T* __restrict__ X, int n_tiles, int sweeps, int d, const double* __restrict__ coef,
                 const float* __restrict__ y, const uint8_t* __restrict__ mask, int keep, float* __restrict__ yhat,
                 double* __restrict__ part) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const uint32_t sbase = smem_u32(smem_raw);
  const uint32_t bar_full = sbase + kTmOffBar, bar_empty = bar_full + 8 * kTmStages;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  constexpr int RPI = 32 / LPR, kSweepRows = kTmWarps * RPI;
  const int tile_rows = sweeps * kSweepRows;
  const uint32_t pitch = (uint32_t)d * sizeof(T);
  const bool has_mask = mask != nullptr, has_y = y != nullptr;
  ring_init<kTmStages>(bar_full, bar_empty, kTmWarps);

  __shared__ double red[kTmWarps][kNStats];
  if (warp == kTmWarps) {
    if (lane == 0)
      ring_produce<kTmStages>(bar_full, bar_empty, n_tiles, tile_rows, X, pitch, sbase, kTmXStage, has_y, y,
                              sbase + kTmOffY, kTmYStage, false, nullptr, 0u, 0u);
  } else {
    // LPR lanes per row, RPI rows per warp iteration: lane (g, j) = (lane / LPR, lane % LPR) reads the 4-feature chunks
    // kk * LPR + j of row g, kk = (k + g) mod 4 for k = 0..3 -- the rotation by g keeps the rows of one shared-memory
    // wavefront on different banks when the row pitch is 128 or 256 bytes.
    const int g = lane / LPR, j = lane % LPR;
    double cf[4][4];
    bool col_ok[4];
    uint32_t coff[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int c = ((k + g) & 3) * LPR + j;
      const int f0 = 4 * c;
      col_ok[k] = f0 < d;
      coff[k] = (uint32_t)c * 4u * (uint32_t)sizeof(T);
#pragma unroll
      for (int e = 0; e < 4; ++e) cf[k][e] = (f0 + e < d) ? coef[f0 + e] : 0.0;
    }
    const double b0 = coef[kMaxD];
    RowStats st;
    // the statistics of a row cost ~25 fp64 instructions: lane (g, j) keeps the row of iteration j (mod LPR) and all 32
    // lanes update their statistics together once per LPR iterations
    double p_keep = 0.0;
    float y_keep = 0.f;
    bool have = false;
    int it8 = 0;
    int s = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
      const int64_t row0 = (int64_t)tile * tile_rows;
      unsigned use_bits = 0xfu;
      if (has_mask) {
        use_bits = 0u;
#pragma unroll
        for (int sw = 0; sw < kTmMaxSweeps; ++sw)
          if (sw < sweeps)
            use_bits |= (__ldg(mask + row0 + sw * kSweepRows + warp * RPI + g) == (uint8_t)keep ? 1u : 0u) << sw;
      }
      mbar_wait(bar_full + 8 * s, phase);
      const uint32_t xs = sbase + s * kTmXStage, ys = sbase + kTmOffY + s * kTmYStage;
      for (int sw = 0; sw < sweeps; ++sw) {
        const int r = sw * kSweepRows + warp * RPI + g;                 // this lane group's row inside the tile
        const bool use = (use_bits >> sw) & 1u;
        const uint32_t row_addr = xs + (uint32_t)r * pitch;
        float x[4][4];
#pragma unroll
        for (int k = 0; k < 4; ++k) lds_row4<T>(row_addr + coff[k], use && col_ok[k], x[k]);
        double a0 = (double)x[0][0] * cf[0][0], a1 = (double)x[2][0] * cf[2][0];   // two chains for latency
#pragma unroll
        for (int e = 1; e < 4; ++e) { a0 = fma((double)x[0][e], cf[0][e], a0); a1 = fma((double)x[2][e], cf[2][e], a1); }
#pragma unroll
        for (int e = 0; e < 4; ++e) { a0 = fma((double)x[1][e], cf[1][e], a0); a1 = fma((double)x[3][e], cf[3][e], a1); }
        double a = a0 + a1;
#pragma unroll
        for (int o = LPR / 2; o >= 1; o >>= 1) a += shfl_xor_d(a, o);
        const double pr = a + b0;
        if (yhat != nullptr && j == 0) yhat[row0 + r] = use ? (float)pr : 0.f;
        if (has_y) {
          if (j == it8 && use) {
            p_keep = pr;
            y_keep = ld_shared_f32(ys + 4u * (uint32_t)r);
            have = true;
          }
          if (++it8 == LPR) {
            if (have) st.add((double)y_keep, p_keep);
            have = false;
            it8 = 0;
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_empty + 8 * s);
      if (++s == kTmStages) { s = 0; phase ^= 1u; }
    }
    if (have) st.add((double)y_keep, p_keep);
    double v[kNStats];
    st.values(v);
    stats_butterfly<1>(v);
    stats_store(red, warp, lane, v);
  }
  stats_fold<kTmWarps>(red, part);
}

// ---- narrow rows (D <= 16): one lane per row behind the same bulk-copy ring ---------------------------------------
// The warp-per-row kernels above leave 31 of 32 lanes idle at the reference's own shape (one feature,
// stage_1_train_model.py:95).  Here a lane owns a row: d conversions + d DFMAs, the statistics of 32 rows per warp
// instruction, yhat written 128 bytes per warp.  fp64-pipe bound at D = 1 (8 bytes per row), HBM-bound from D = 4.
constexpr int kSnStages = 6;
constexpr int kSnWarps = 7;                        // consumer warps (+ 1 producer warp = 256 threads, 2 CTAs per SM)
constexpr int kSnConsumers = 32 * kSnWarps;
constexpr int kSnThreads = kSnConsumers + 32;

template <int DP>
struct SnGeom {
  static constexpr int RPT = DP <= 2 ? 4 : (DP == 4 ? 2 : 1);   // rows per lane per stage
  static constexpr int kRows = kSnConsumers * RPT;
  static constexpr uint32_t kXStage = kRows * DP * 4;            // sized for fp32
  static constexpr uint32_t kYStage = kRows * 4;
  static constexpr uint32_t kMStage = kRows;
  static constexpr uint32_t kOffY = kSnStages * kXStage;
  static constexpr uint32_t kOffM = kOffY + kSnStages * kYStage;
  static constexpr uint32_t kOffBar = kOffM + kSnStages * kMStage;
  static constexpr uint32_t kSmem = kOffBar + 2 * kSnStages * 8 + 128;
};

// PLAIN: the metrics-only pass over unmasked rows (no row mask, no prediction store, labels present) -- the selects, the
// mask load and the predicated store of the general flavour compile away (they were a quarter of its instructions).
template <typename T, int DP, bool EXACT, bool PLAIN>
__global__ void __launch_bounds__(kSnThreads, 2)
score_narrow_kernel(const T* __restrict__ X, int n_tiles, int d, const double* __restrict__ coef,
                    const float* __restrict__ y, const uint8_t* __restrict__ mask_arg, int keep, float* __restrict__ yhat_arg,
                    double* __restrict__ part) {
  const uint8_t* mask = PLAIN ? nullptr : mask_arg;
  float* yhat = PLAIN ? nullptr : yhat_arg;
  using G = SnGeom<DP>;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const uint32_t sbase = smem_u32(smem_raw);
  const uint32_t bar_full = sbase + G::kOffBar, bar_empty = bar_full + 8 * kSnStages;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool has_mask = mask != nullptr, has_y = PLAIN || y != nullptr;
  const uint32_t row_bytes = (uint32_t)d * sizeof(T);
  ring_init<kSnStages>(bar_full, bar_empty, kSnWarps);
  __shared__ double red[kSnWarps][kNStats];
  if (warp == kSnWarps) {
    if (lane == 0)
      ring_produce<kSnStages>(bar_full, bar_empty, n_tiles, G::kRows, X, row_bytes, sbase, G::kXStage, has_y, y,
                              sbase + G::kOffY, G::kYStage, has_mask, mask, sbase + G::kOffM, G::kMStage);
  } else {
    double cf[DP];
#pragma unroll
    for (int k = 0; k < DP; ++k) cf[k] = k < d ? coef[k] : 0.0;
    const double b0 = coef[kMaxD];
    RowStats st;
    int s = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
      mbar_wait(bar_full + 8 * s, phase);
      const uint32_t xs = sbase + s * G::kXStage, ys = sbase + G::kOffY + s * G::kYStage, ms = sbase + G::kOffM + s * G::kMStage;
      const int64_t row0 = (int64_t)tile * G::kRows;
      // all rows of this lane first (loads, dot products, prediction store), then the statistics of all of them without
      // control flow in between: the fp64 / conversion chains of the RPT rows interleave (the kernel was issue- and
      // dependency-bound at D = 1)
      float yv[G::RPT];
      double pr[G::RPT];
      bool use[G::RPT];
      bool fast = true;
#pragma unroll
      for (int rr = 0; rr < G::RPT; ++rr) {
        const int r = rr * kSnConsumers + threadIdx.x;          // consecutive lanes, consecutive rows
        use[rr] = !has_mask || ld_shared_u8(ms + (uint32_t)r) == (uint32_t)keep;
        float x[DP];
        if constexpr (EXACT) ld_vals_vec<T, DP>(xs + (uint32_t)r * row_bytes, x);
        else ld_vals_any<T, DP>(xs + (uint32_t)r * row_bytes, 0, d, x);
        double a0 = b0, a1 = 0.0;                                // two chains
#pragma unroll
        for (int k = 0; k < DP; k += 2) {
          a0 = fma((double)x[k], cf[k], a0);
          if (k + 1 < DP) a1 = fma((double)x[k + 1], cf[k + 1], a1);
        }
        pr[rr] = DP > 1 ? a0 + a1 : a0;
        if (yhat != nullptr) yhat[row0 + r] = use[rr] ? (float)pr[rr] : 0.f;
        yv[rr] = has_y ? ld_shared_f32(ys + 4u * (uint32_t)r) : 1.f;
        const float ayf = fabsf(yv[rr]);
        fast = fast && (!use[rr] || (ayf > 1e-30f && ayf < 1e30f));
      }
      if (has_y) {
        if (__all_sync(0xffffffffu, fast)) {
#pragma unroll
          for (int rr = 0; rr < G::RPT; ++rr) st.add_fast(yv[rr], pr[rr], use[rr]);
        } else {                                                 // a zero / huge label somewhere in the warp: exact path
#pragma unroll
          for (int rr = 0; rr < G::RPT; ++rr)
            if (use[rr]) st.add((double)yv[rr], pr[rr]);
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_empty + 8 * s);
      if (++s == kSnStages) { s = 0; phase ^= 1u; }
    }
    double v[kNStats];
    st.values(v);
    stats_butterfly<1>(v);
    stats_store(red, warp, lane, v);
  }
  stats_fold<kSnWarps>(red, part);
}

// ---- model_metrics on two vectors (stage_1_train_model.py:79-90): no X, no dot product -- the statistics alone, on
// fp32 or fp64 inputs (the reference computes them on float64 arrays; b2_metrics(B2_F64) matches it to rounding) -----
template <typename V>
__global__ void __launch_bounds__(kScoreThreads)
metrics_kernel(const V* __restrict__ ya, const V* __restrict__ yp, int64_t n, double* __restrict__ part) {
  RowStats st;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) st.add_exact((double)ya[i], (double)yp[i]);
  double v[kNStats];
  st.values(v);
  __shared__ double red[kScoreWarps][kNStats];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  stats_butterfly<1>(v);
  stats_store(red, warp, lane, v);
  stats_fold<kScoreWarps>(red, part);
}

// ---- residual gradient of the refined fit (b2_fit_refined; DESIGN.md section 2) -----------------------------------------
// The model is yhat = b0' + (x - m).beta (st: ctx->refine).  Per kept row e = y - b0' - (x - m).beta, and the pass sums
// g_j = sum (x_j - m_j) e, g_1 = sum e and sum e^2 (the last read only by b2_residual_moments), everything in fp64 from the
// exactly converted x: e is a small difference of large terms.  The three layouts of scoring carry it: register-fed (any layout, the tails), the TMA ring (wide contiguous
// rows), one lane per row (d <= 16).  A lane keeps the fp64 sums of the features it loads.  A dropped row gets x = 0 and
// e = 0 by selects, so whatever it holds never reaches a sum.  Each CTA combines its sums in a fixed order into
// part[blockIdx.x][kGradOut] (features, then g_1 at kMaxD, sum e^2 at kMaxD + 1); the ordered reduce adds the CTAs in order.
template <typename T>
__device__ __forceinline__ float ld_x_f32(const T* __restrict__ p);
template <>
__device__ __forceinline__ float ld_x_f32<float>(const float* __restrict__ p) { return __ldg(p); }
template <>
__device__ __forceinline__ float ld_x_f32<__nv_bfloat16>(const __nv_bfloat16* __restrict__ p) { return __bfloat162float(*p); }

// register-fed: one warp per row, four rows in flight; lane features lane * 4 + k (vec) or lane + 32 k
template <typename T>
__global__ void __launch_bounds__(kScoreThreads)
grad_kernel(const T* __restrict__ X, int64_t n, int d, int64_t ldx, const double* __restrict__ st,
            const float* __restrict__ y, const uint8_t* __restrict__ mask, int keep, int vec, double* __restrict__ part) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double cf[4], mv[4], acc[4], acc1 = 0.0, acc2 = 0.0;
  int fj[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    fj[k] = vec ? lane * 4 + k : lane + 32 * k;
    cf[k] = fj[k] < d ? st[kRfBeta + fj[k]] : 0.0;
    mv[k] = fj[k] < d ? st[kRfMean + fj[k]] : 0.0;
    acc[k] = 0.0;
  }
  const double b0 = st[kRfB0];
  const int64_t warps_total = (int64_t)gridDim.x * kScoreWarps;
  const int64_t gw = (int64_t)blockIdx.x * kScoreWarps + warp;
  constexpr int kU = 4;
  for (int64_t base = gw * kU; base < n; base += warps_total * kU) {
    float x[kU][4];
    bool use[kU];
#pragma unroll
    for (int u = 0; u < kU; ++u) {
      const int64_t row = base + u;
      use[u] = row < n;
      if (use[u] && mask != nullptr) use[u] = (__ldg(mask + row) == (uint8_t)keep);
#pragma unroll
      for (int k = 0; k < 4; ++k) x[u][k] = 0.f;
      const T* xr = X + row * ldx;
      if (use[u]) {
        if (vec) {
          if (lane * 4 < d) {
            if constexpr (sizeof(T) == 4) {
              const float4 v = __ldg(reinterpret_cast<const float4*>(xr) + lane);
              x[u][0] = v.x; x[u][1] = v.y; x[u][2] = v.z; x[u][3] = v.w;
            } else {
              const uint2 v = __ldg(reinterpret_cast<const uint2*>(xr) + lane);
              x[u][0] = __uint_as_float(v.x << 16); x[u][1] = __uint_as_float(v.x & 0xffff0000u);
              x[u][2] = __uint_as_float(v.y << 16); x[u][3] = __uint_as_float(v.y & 0xffff0000u);
            }
          }
        } else {
#pragma unroll
          for (int k = 0; k < 4; ++k)
            if (fj[k] < d) x[u][k] = ld_x_f32<T>(xr + fj[k]);
        }
      }
    }
    double dot[kU];
#pragma unroll
    for (int u = 0; u < kU; ++u) {
      double a = 0.0;
#pragma unroll
      for (int k = 0; k < 4; ++k) a = fma((double)x[u][k] - mv[k], cf[k], a);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) a += shfl_xor_d(a, o);   // every lane ends with the same sum (a + b == b + a)
      dot[u] = a;
    }
#pragma unroll
    for (int u = 0; u < kU; ++u) {
      const float yv = use[u] ? __ldg(y + base + u) : 0.f;
      const double e = use[u] ? ((double)yv - b0) - dot[u] : 0.0;
#pragma unroll
      for (int k = 0; k < 4; ++k) acc[k] = fma((double)x[u][k] - mv[k], e, acc[k]);
      acc1 += e;
      acc2 = fma(e, e, acc2);
    }
  }
  __shared__ double red[kScoreWarps][kGradOut];
#pragma unroll
  for (int k = 0; k < 4; ++k)
    if (fj[k] < d) red[warp][fj[k]] = acc[k];
  if (lane == 0) {
    red[warp][kMaxD] = acc1;
    red[warp][kMaxD + 1] = acc2;
  }
  grad_fold<kScoreWarps>(red, d, part);
}

// TMA ring: the producer and the lane layout of score_tma_kernel; the labels are always streamed.  beta and the sums stay in
// registers, m is read from shared memory (two 16-byte loads per chunk): all three in registers spill at 128 per thread.
template <typename T, int LPR>
__global__ void __launch_bounds__(kTmThreads, 1)
grad_tma_kernel(const T* __restrict__ X, int n_tiles, int sweeps, int d, const double* __restrict__ st,
                const float* __restrict__ y, const uint8_t* __restrict__ mask, int keep, double* __restrict__ part) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const uint32_t sbase = smem_u32(smem_raw);
  const uint32_t bar_full = sbase + kTmOffBar, bar_empty = bar_full + 8 * kTmStages;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  constexpr int RPI = 32 / LPR, kSweepRows = kTmWarps * RPI;
  const int tile_rows = sweeps * kSweepRows;
  const uint32_t pitch = (uint32_t)d * sizeof(T);
  ring_init<kTmStages>(bar_full, bar_empty, kTmWarps);

  __shared__ double red[kTmWarps][kGradOut];
  __shared__ __align__(16) double m_s[kMaxD];
  __shared__ double e2_s[kTmWarps][32];   // sum e^2 of the row group whose first lane this is: a register would spill
  for (int f = threadIdx.x; f < kMaxD; f += blockDim.x) m_s[f] = f < d ? st[kRfMean + f] : 0.0;
  for (int t = threadIdx.x; t < kTmWarps * 32; t += blockDim.x) e2_s[t / 32][t % 32] = 0.0;
  __syncthreads();
  if (warp == kTmWarps) {
    if (lane == 0)
      ring_produce<kTmStages>(bar_full, bar_empty, n_tiles, tile_rows, X, pitch, sbase, kTmXStage, true, y,
                              sbase + kTmOffY, kTmYStage, false, nullptr, 0u, 0u);
  } else {
    const int g = lane / LPR, j = lane % LPR;
    double cf[4][4], acc[4][4];
    bool col_ok[4];
    uint32_t coff[4];
    int f0[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int c = ((k + g) & 3) * LPR + j;
      f0[k] = 4 * c;
      col_ok[k] = f0[k] < d;
      coff[k] = (uint32_t)c * 4u * (uint32_t)sizeof(T);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int f = f0[k] + e;
        cf[k][e] = f < d ? st[kRfBeta + f] : 0.0;
        acc[k][e] = 0.0;
      }
    }
    const double b0 = st[kRfB0];
    double acc1 = 0.0;
    int s = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
      const int64_t row0 = (int64_t)tile * tile_rows;
      unsigned use_bits = 0xfu;
      if (mask != nullptr) {
        use_bits = 0u;
#pragma unroll
        for (int sw = 0; sw < kTmMaxSweeps; ++sw)
          if (sw < sweeps)
            use_bits |= (__ldg(mask + row0 + sw * kSweepRows + warp * RPI + g) == (uint8_t)keep ? 1u : 0u) << sw;
      }
      mbar_wait(bar_full + 8 * s, phase);
      const uint32_t xs = sbase + s * kTmXStage, ys = sbase + kTmOffY + s * kTmYStage;
      for (int sw = 0; sw < sweeps; ++sw) {
        const int r = sw * kSweepRows + warp * RPI + g;
        const bool use = (use_bits >> sw) & 1u;
        const uint32_t row_addr = xs + (uint32_t)r * pitch;
        float x[4][4];
#pragma unroll
        for (int k = 0; k < 4; ++k) lds_row4<T>(row_addr + coff[k], use && col_ok[k], x[k]);
        double v[4][4];                                                // x - m, exact inputs, one fp64 rounding
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const double2 m01 = *reinterpret_cast<const double2*>(&m_s[f0[k] & (kMaxD - 1)]);
          const double2 m23 = *reinterpret_cast<const double2*>(&m_s[(f0[k] & (kMaxD - 1)) + 2]);
          v[k][0] = (double)x[k][0] - m01.x; v[k][1] = (double)x[k][1] - m01.y;
          v[k][2] = (double)x[k][2] - m23.x; v[k][3] = (double)x[k][3] - m23.y;
        }
        double a0 = 0.0, a1 = 0.0;                                     // two chains for latency
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          a0 = fma(v[0][e], cf[0][e], a0);
          a1 = fma(v[2][e], cf[2][e], a1);
        }
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          a0 = fma(v[1][e], cf[1][e], a0);
          a1 = fma(v[3][e], cf[3][e], a1);
        }
        double a = a0 + a1;
#pragma unroll
        for (int o = LPR / 2; o >= 1; o >>= 1) a += shfl_xor_d(a, o);
        const float yv = use ? ld_shared_f32(ys + 4u * (uint32_t)r) : 0.f;
        const double e = use ? ((double)yv - b0) - a : 0.0;
#pragma unroll
        for (int k = 0; k < 4; ++k)
#pragma unroll
          for (int q = 0; q < 4; ++q) acc[k][q] = fma(v[k][q], e, acc[k][q]);
        if (j == 0) {
          acc1 += e;
          e2_s[warp][lane] = fma(e, e, e2_s[warp][lane]);
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_empty + 8 * s);
      if (++s == kTmStages) { s = 0; phase ^= 1u; }
    }
    // the row groups of a warp hold the same features (rotated): they add into red[warp] one group after the other
#pragma unroll 1
    for (int gg = 0; gg < RPI; ++gg) {
      if (g == gg) {
#pragma unroll
        for (int k = 0; k < 4; ++k)
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const int f = f0[k] + q;
            if (f < d) red[warp][f] = gg == 0 ? acc[k][q] : red[warp][f] + acc[k][q];
          }
        if (j == 0) {
          red[warp][kMaxD] = gg == 0 ? acc1 : red[warp][kMaxD] + acc1;
          red[warp][kMaxD + 1] = gg == 0 ? e2_s[warp][lane] : red[warp][kMaxD + 1] + e2_s[warp][lane];
        }
      }
      __syncwarp();
    }
  }
  grad_fold<kTmWarps>(red, d, part);
}

// narrow rows (d <= 16): one lane per row behind the bulk-copy ring of score_narrow_kernel
template <typename T, int DP, bool EXACT>
__global__ void __launch_bounds__(kSnThreads, DP >= 16 ? 1 : 2)   // 16 features: 3 x 16 doubles per lane need > 128 registers
grad_narrow_kernel(const T* __restrict__ X, int n_tiles, int d, const double* __restrict__ st, const float* __restrict__ y,
                   const uint8_t* __restrict__ mask, int keep, double* __restrict__ part) {
  using G = SnGeom<DP>;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const uint32_t sbase = smem_u32(smem_raw);
  const uint32_t bar_full = sbase + G::kOffBar, bar_empty = bar_full + 8 * kSnStages;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool has_mask = mask != nullptr;
  const uint32_t row_bytes = (uint32_t)d * sizeof(T);
  ring_init<kSnStages>(bar_full, bar_empty, kSnWarps);
  __shared__ double red[kSnWarps][kGradOut];
  if (warp == kSnWarps) {
    if (lane == 0)
      ring_produce<kSnStages>(bar_full, bar_empty, n_tiles, G::kRows, X, row_bytes, sbase, G::kXStage, true, y,
                              sbase + G::kOffY, G::kYStage, has_mask, mask, sbase + G::kOffM, G::kMStage);
  } else {
    double cf[DP], mv[DP], acc[DP];
#pragma unroll
    for (int k = 0; k < DP; ++k) {
      cf[k] = k < d ? st[kRfBeta + k] : 0.0;
      mv[k] = k < d ? st[kRfMean + k] : 0.0;
      acc[k] = 0.0;
    }
    const double b0 = st[kRfB0];
    double acc1 = 0.0, acc2 = 0.0;
    int s = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
      mbar_wait(bar_full + 8 * s, phase);
      const uint32_t xs = sbase + s * G::kXStage, ys = sbase + G::kOffY + s * G::kYStage, ms = sbase + G::kOffM + s * G::kMStage;
#pragma unroll
      for (int rr = 0; rr < G::RPT; ++rr) {
        const int r = rr * kSnConsumers + threadIdx.x;
        const bool use = !has_mask || ld_shared_u8(ms + (uint32_t)r) == (uint32_t)keep;
        float x[DP];
        if constexpr (EXACT) ld_vals_vec<T, DP>(xs + (uint32_t)r * row_bytes, x);
        else ld_vals_any<T, DP>(xs + (uint32_t)r * row_bytes, 0, d, x);
#pragma unroll
        for (int k = 0; k < DP; ++k) x[k] = use ? x[k] : 0.f;
        double a0 = 0.0, a1 = 0.0;
#pragma unroll
        for (int k = 0; k < DP; k += 2) {
          a0 = fma((double)x[k] - mv[k], cf[k], a0);
          if (k + 1 < DP) a1 = fma((double)x[k + 1] - mv[k + 1], cf[k + 1], a1);
        }
        const float yv = use ? ld_shared_f32(ys + 4u * (uint32_t)r) : 0.f;
        const double e = use ? ((double)yv - b0) - (a0 + a1) : 0.0;
#pragma unroll
        for (int k = 0; k < DP; ++k) acc[k] = fma((double)x[k] - mv[k], e, acc[k]);
        acc1 += e;
        acc2 = fma(e, e, acc2);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_empty + 8 * s);
      if (++s == kSnStages) { s = 0; phase ^= 1u; }
    }
#pragma unroll
    for (int k = 0; k <= DP + 1; ++k) {
      double v = k < DP ? acc[k] : (k == DP ? acc1 : acc2);
#pragma unroll
      for (int o = 16; o >= 1; o >>= 1) v += shfl_xor_d(v, o);
      if (lane == 0) {
        if (k < DP && k < d) red[warp][k] = v;
        if (k >= DP) red[warp][kMaxD + k - DP] = v;
      }
    }
  }
  grad_fold<kSnWarps>(red, d, part);
}

// launch_ordered_reduce: one thread per entry, eight loads in flight, the combines in CTA order
__global__ void ordered_reduce_kernel(const double* __restrict__ part, int stride, int n_ctas, int first, int n_lin,
                                      unsigned max_mask, int d1, int tri_off, int tri_pitch, double* __restrict__ acc) {
  const int total = n_lin + d1 * d1;
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < total; e += gridDim.x * blockDim.x) {
    int off = e;
    if (e >= n_lin) {
      const int q = e - n_lin, i = q / d1, j = q - i * d1;
      if (i > j) continue;
      off = tri_off + i * tri_pitch + j;
    }
    const bool is_max = e < n_lin && e < 32 && ((max_mask >> e) & 1u) != 0;
    double v = first ? 0.0 : acc[off];
    int c = 0;
    for (; c + 8 <= n_ctas; c += 8) {
      double p[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) p[u] = part[(size_t)(c + u) * stride + off];
#pragma unroll
      for (int u = 0; u < 8; ++u) v = is_max ? fmax(v, p[u]) : v + p[u];
    }
    for (; c < n_ctas; ++c) v = is_max ? fmax(v, part[(size_t)c * stride + off]) : v + part[(size_t)c * stride + off];
    acc[off] = v;
  }
}

// scoring's statistics combine their two maxima (4 and 9) with fmax
constexpr unsigned kStatsMaxMask = (1u << 4) | (1u << 9);

}  // namespace

int launch_ordered_reduce(b2_ctx* ctx, const double* part, int stride, int n_ctas, bool first, int n_lin,
                          unsigned max_mask, double* acc, int d1, int tri_off, int tri_pitch) {
  B2_CUDA(cudaGetLastError());
  const int total = n_lin + d1 * d1;
  ordered_reduce_kernel<<<(total + 255) / 256, 256, 0, ctx->stream>>>(part, stride, n_ctas, first ? 1 : 0, n_lin,
                                                                      max_mask, d1, tri_off, tri_pitch, acc);
  B2_CUDA(cudaGetLastError());
  ctx->launches += 2;
  return B2_OK;
}

RowPlan plan_rows(const b2_ctx* ctx, const void* X, int x_dtype, int64_t n, int d, int64_t ldx, const float* y,
                  const uint8_t* mask) {
  RowPlan p;
  const int es = x_dtype == B2_F32 ? 4 : 2;
  auto aligned16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  const bool ring_rows = ldx == d && aligned16(X) && (y == nullptr || aligned16(y));
  int tile_rows = 0, cap = 0;
  if (ring_rows && d <= 16 && (mask == nullptr || aligned16(mask))) {
    p.kind = RowPlan::kNarrow;
    p.dp = narrow_dp(d);
    tile_rows = with_int<1, 2, 4, 8, 16>(p.dp, [](auto DP) { return SnGeom<decltype(DP)::value>::kRows; });
    cap = ctx->sm_count * 2;
  } else if (ring_rows && d > 16 && d % 4 == 0 && (d * es) % 16 == 0) {
    p.kind = RowPlan::kWide;
    p.lpr = d <= 32 ? 2 : (d <= 64 ? 4 : 8);                     // lanes per row: 4 chunks of 4 features per lane
    const int sweep_rows = kTmWarps * (32 / p.lpr);
    p.sweeps = (int)(kTmXStage / (uint32_t)(sweep_rows * d * es));
    if (p.sweeps > kTmTileRowsMax / sweep_rows) p.sweeps = kTmTileRowsMax / sweep_rows;
    tile_rows = p.sweeps * sweep_rows;
    cap = ctx->sm_count;
  }
  const int64_t n_tiles = tile_rows > 0 ? n / tile_rows : 0;
  if (n_tiles > 0 && n_tiles <= 0x7fffffff) {
    p.n_tiles = (int)n_tiles;
    p.grid = p.n_tiles < cap ? p.n_tiles : cap;
    p.done = n_tiles * tile_rows;
  }
  p.direct = p.done < n || n == 0;
  p.rest = n - p.done;
  const uintptr_t x_rest = reinterpret_cast<uintptr_t>(X) + (size_t)p.done * ldx * es;
  p.vec = (d % 4 == 0) && ((ldx * es) % (4 * es) == 0) && (x_rest % (4 * es) == 0);
  int64_t want = (p.rest + kScoreWarps * 4 - 1) / (kScoreWarps * 4);
  if (want < 1) want = 1;
  p.direct_grid = (int)(want < ctx->score_ctas ? want : ctx->score_ctas);
  return p;
}

int launch_metrics(b2_ctx* ctx, const void* y, const void* yhat, int dtype, int64_t n, bool first) {
  int64_t want = (n + kScoreThreads * 8 - 1) / (kScoreThreads * 8);
  if (want < 1) want = 1;
  const int grid = (int)(want < ctx->score_ctas ? want : ctx->score_ctas);
  if (dtype == B2_F32)
    metrics_kernel<float><<<grid, kScoreThreads, 0, ctx->stream>>>(static_cast<const float*>(y), static_cast<const float*>(yhat),
                                                                   n, ctx->score_part);
  else
    metrics_kernel<double><<<grid, kScoreThreads, 0, ctx->stream>>>(static_cast<const double*>(y),
                                                                    static_cast<const double*>(yhat), n, ctx->score_part);
  return launch_ordered_reduce(ctx, ctx->score_part, kNStats, grid, first, kNStats, kStatsMaxMask, score_totals(ctx));
}

int launch_score(b2_ctx* ctx, const void* X, int x_dtype, int64_t n, int d, int64_t ldx, const float* y,
                 const uint8_t* mask, int keep, float* yhat, bool first_block) {
  const RowPlan p = plan_rows(ctx, X, x_dtype, n, d, ldx, y, mask);
  if (p.n_tiles > 0) {
    const int rc = with_rows(x_dtype, X, [&](auto* Xr) {
      using T = row_t<decltype(Xr)>;
      if (p.kind == RowPlan::kWide)
        return with_int<2, 4, 8>(p.lpr, [&](auto LPR) {
          return launch_smem(score_tma_kernel<T, decltype(LPR)::value>, p.grid, kTmThreads, kTmSmem, ctx->stream, Xr,
                             p.n_tiles, p.sweeps, d, ctx->coef_dev, y, mask, keep, yhat, ctx->score_part);
        });
      return with_int<1, 2, 4, 8, 16>(p.dp, [&](auto DP) {
        constexpr int kDP = decltype(DP)::value;
        const bool plain = mask == nullptr && yhat == nullptr && y != nullptr;
        auto kernel = d != kDP ? score_narrow_kernel<T, kDP, false, false>
                    : plain    ? score_narrow_kernel<T, kDP, true, true> : score_narrow_kernel<T, kDP, true, false>;
        return launch_smem(kernel, p.grid, kSnThreads, SnGeom<kDP>::kSmem, ctx->stream, Xr, p.n_tiles, d, ctx->coef_dev,
                           y, mask, keep, yhat, ctx->score_part);
      });
    });
    if (rc != B2_OK) return rc;
    if (int r = launch_ordered_reduce(ctx, ctx->score_part, kNStats, p.grid, first_block, kNStats, kStatsMaxMask,
                                     score_totals(ctx)))
      return r;
    first_block = false;
  }
  if (!p.direct) return B2_OK;
  const int es = x_dtype == B2_F32 ? 4 : 2;
  const char* Xt = static_cast<const char*>(X) + (size_t)p.done * ldx * es;
  const float* yt = y != nullptr ? y + p.done : nullptr;
  const uint8_t* mt = mask != nullptr ? mask + p.done : nullptr;
  float* yhat_t = yhat != nullptr ? yhat + p.done : nullptr;
  const bool rows16 = p.vec && ((ldx * es) % 16 == 0) && ((reinterpret_cast<uintptr_t>(Xt) & 15) == 0 || x_dtype != B2_F32);
  with_rows(x_dtype, Xt, [&](auto* Xr) {
    using T = row_t<decltype(Xr)>;
    if (rows16)
      score_kernel_rows8<T><<<p.direct_grid, kScoreThreads, 0, ctx->stream>>>(Xr, p.rest, d, ldx, ctx->coef_dev, yt, mt,
                                                                               keep, yhat_t, ctx->score_part);
    else
      score_kernel<T><<<p.direct_grid, kScoreThreads, 0, ctx->stream>>>(Xr, p.rest, d, ldx, ctx->coef_dev, yt, mt, keep,
                                                                         yhat_t, p.vec, ctx->score_part);
    return B2_OK;
  });
  return launch_ordered_reduce(ctx, ctx->score_part, kNStats, p.direct_grid, first_block, kNStats, kStatsMaxMask,
                               score_totals(ctx));
}

// The residual gradient over the rows [0, n): the kernels of launch_score's plan (the labels are always present).
int launch_grad(b2_ctx* ctx, const void* X, int x_dtype, int64_t n, int d, int64_t ldx, const float* y,
                const uint8_t* mask, int keep, bool first_block) {
  const RowPlan p = plan_rows(ctx, X, x_dtype, n, d, ldx, y, mask);
  if (p.n_tiles > 0) {
    const int rc = with_rows(x_dtype, X, [&](auto* Xr) {
      using T = row_t<decltype(Xr)>;
      if (p.kind == RowPlan::kWide)
        return with_int<2, 4, 8>(p.lpr, [&](auto LPR) {
          return launch_smem(grad_tma_kernel<T, decltype(LPR)::value>, p.grid, kTmThreads, kTmSmem, ctx->stream, Xr,
                             p.n_tiles, p.sweeps, d, ctx->refine, y, mask, keep, ctx->grad_part);
        });
      return with_int<1, 2, 4, 8, 16>(p.dp, [&](auto DP) {
        constexpr int kDP = decltype(DP)::value;
        auto kernel = d == kDP ? grad_narrow_kernel<T, kDP, true> : grad_narrow_kernel<T, kDP, false>;
        return launch_smem(kernel, p.grid, kSnThreads, SnGeom<kDP>::kSmem, ctx->stream, Xr, p.n_tiles, d, ctx->refine, y,
                           mask, keep, ctx->grad_part);
      });
    });
    if (rc != B2_OK) return rc;
    if (int r = launch_ordered_reduce(ctx, ctx->grad_part, kGradOut, p.grid, first_block, kGradOut, 0u,
                                     ctx->refine + kRfGrad))
      return r;
    first_block = false;
  }
  if (!p.direct) return B2_OK;
  const int es = x_dtype == B2_F32 ? 4 : 2;
  const char* Xt = static_cast<const char*>(X) + (size_t)p.done * ldx * es;
  const uint8_t* mt = mask != nullptr ? mask + p.done : nullptr;
  with_rows(x_dtype, Xt, [&](auto* Xr) {
    using T = row_t<decltype(Xr)>;
    grad_kernel<T><<<p.direct_grid, kScoreThreads, 0, ctx->stream>>>(Xr, p.rest, d, ldx, ctx->refine, y + p.done, mt, keep,
                                                                      p.vec, ctx->grad_part);
    return B2_OK;
  });
  return launch_ordered_reduce(ctx, ctx->grad_part, kGradOut, p.direct_grid, first_block, kGradOut, 0u,
                               ctx->refine + kRfGrad);
}

}  // namespace b2
