// glm.cu -- the row passes of the generalised linear regressors (b2_glm_pass, b2_glm_line_search, b2_glm_predict;
// DESIGN.md section 10) and of binary logistic regression (b2_logistic_*, b2_label_scan; DESIGN.md section 11).
//
// scikit-learn's Newton solver (solver="newton-cholesky") needs, at the coefficients w, b of each iteration and with
// eta = x.w + b per kept row, the half-Tweedie loss, its gradient g and Hessian h (loss(y, eta) and its derivatives in
// eta, the Cython formulas of sklearn/_loss/_loss.pyx.tp branch by branch), and from them
//   sum loss, sum g [x 1] (HBM-bound) and sum |h| [x 1][x 1]^T (2 (D + 1)^2 flops per row: fp64-compute bound).
// One pass per call over 32-row tiles:
//   (1) the tile -> shared memory as z = [x 1] in fp64 from the stored value (exact), zero for rows not kept;
//   (2) eta (and, for the line search, deta = x.step + db) per row: the lanes of a warp over the features, a butterfly;
//   (3) loss, g, h (or the loss at eta + t deta for t = 1, 1/2, ..., one step per lane) per kept row, by selects;
//   (4) the gradient: thread j adds g_r z_rj over the tile's rows in order;
//   (5) the Hessian on the fp64 tensor core (mma.sync m8n8k4 f64) with the upper-block schedule (b2_dmma.cuh): A =
//       the |h|-scaled rows, B = the rows, K = the 32 rows of the tile.  The (D + 1)^2 output is cut in 16 x 16 blocks;
//       only blocks on or above the diagonal are computed, each warp holding up to six of them in registers for the
//       whole launch (4 DMMAs per 2 + 2 fragment loads), the 8 x 8 tile below the diagonal of a diagonal block skipped:
//       153 of the 289 8 x 8 tiles at D = 128.
// The rows take scoring's plan (plan_rows): contiguous 16-byte aligned rows stream through the bulk-copy ring in whole
// tiles, the rest (and every other layout) is read by the same consumers from global memory.  Each CTA writes its sums
// in a fixed order, the ordered reduce adds the CTAs in order: two calls return identical sums.
#include "b2_internal.cuh"
#include "b2_dmma.cuh"

namespace b2 {
namespace {

constexpr int kGlmBlocks = (kMaxD + 1 + 15) / 16;  // 9 blocks of 16 columns of [x 1]
// 16 x 16 blocks per warp: 6
constexpr int kGlmSB = (kGlmBlocks * (kGlmBlocks + 1) / 2 + kTileWarps - 1) / kTileWarps;

__host__ __device__ inline int glm_dp(int d) { return (d + 1 + 15) & ~15; }   // columns of [x 1], padded to 16
size_t glm_smem_bytes(int dp, bool ring, int mode) {
  const size_t tile = (size_t)kTileRows * tile_vpitch(dp);
  return tile_ring_bytes(ring, true) +
         sizeof(double) * (tile * (mode == kGlmHessian ? 2 : 1) + 3 * kMaxD + 8 + 3 * kTileRows + 2 * kTileWarps * 32) +
         sizeof(int) * kUpperTable;
}

// The pointwise half-Tweedie loss, gradient and Hessian in eta, sklearn's Cython branches: the log link at any power
// (0, 1 and 2 have their own), the identity link at power 0.
__device__ __forceinline__ double glm_loss(int link, double p, double y, double eta) {
  if (link == B2_GLM_IDENTITY) return 0.5 * (eta - y) * (eta - y);
  if (p == 0.0) {
    const double e1 = exp(eta);
    return 0.5 * (e1 - y) * (e1 - y);
  }
  if (p == 1.0) return exp(eta) - y * eta;
  if (p == 2.0) return eta + y * exp(-eta);
  return exp((2.0 - p) * eta) / (2.0 - p) - y * exp((1.0 - p) * eta) / (1.0 - p);
}

__device__ __forceinline__ void glm_point(int link, double p, double y, double eta, double& loss, double& g,
                                          double& h) {
  if (link == B2_GLM_IDENTITY) {
    g = eta - y;
    loss = 0.5 * g * g;
    h = 1.0;
  } else if (p == 0.0) {
    const double e1 = exp(eta);
    loss = 0.5 * (e1 - y) * (e1 - y);
    g = e1 * (e1 - y);
    h = e1 * (2 * e1 - y);
  } else if (p == 1.0) {
    const double e = exp(eta);
    loss = e - y * eta;
    g = e - y;
    h = e;
  } else if (p == 2.0) {
    const double e = exp(-eta);
    loss = eta + y * e;
    g = 1.0 - y * e;
    h = e * y;
  } else {
    const double e1 = exp((1.0 - p) * eta), e2 = exp((2.0 - p) * eta);
    loss = e2 / (2.0 - p) - y * e1 / (1.0 - p);
    g = e2 - y * e1;
    h = (2.0 - p) * e2 - (1.0 - p) * y * e1;
  }
}

// constant_to_optimal_zero(y): the term the loss drops (0 for squared error)
__device__ __forceinline__ double glm_const(int link, double p, double y) {
  if (link == B2_GLM_IDENTITY || p == 0.0) return 0.0;
  if (p == 1.0) return (y == 0.0 ? 0.0 : y * log(y)) - y;          // xlogy(y, y) - y
  if (p == 2.0) return -log(y) - 1.0;
  return pow(fmax(y, 0.0), 2.0 - p) / (1.0 - p) / (2.0 - p);
}

// The half-binomial loss of the logistic fits (sklearn's HalfBinomialLoss), t = 1 for the positive label, 0 otherwise.
// closs_half_binomial: log1pexp(eta) - t eta, log1pexp with sklearn's branches
__device__ __forceinline__ double binom_loss(double t, double eta) {
  double l;
  if (eta <= -37.0) l = exp(eta);
  else if (eta <= -2.0) l = log1p(exp(eta));
  else if (eta <= 18.0) l = log(1.0 + exp(eta));
  else if (eta <= 33.3) l = eta + exp(-eta);
  else l = eta;
  return l - t * eta;
}

// the loss of closs_grad_half_binomial: sklearn's line search evaluates loss_gradient, whose loss is written this way
__device__ __forceinline__ double binom_ladder_loss(double t, double eta) {
  if (eta <= -37.0) return exp(eta) - t * eta;
  if (eta <= -2.0) return log1p(exp(eta)) - t * eta;
  if (eta <= 18.0) return log1p(exp(-eta)) + (1.0 - t) * eta;
  return exp(-eta) + (1.0 - t) * eta;
}

// cgrad_hess_half_binomial: g = expit(eta) - t, h = expit(eta) (1 - expit(eta)), exp(eta) to first order below -37
__device__ __forceinline__ void binom_grad_hess(double t, double eta, double& g, double& h) {
  if (eta > -37.0) {
    const double e = exp(-eta);
    g = ((1.0 - t) - t * e) / (1.0 + e);
    h = e / ((1.0 + e) * (1.0 + e));
  } else {
    const double e = exp(eta);
    g = e - t;
    h = e;
  }
}

// y inside the loss's interval: (-inf, inf) for p <= 0, [0, inf) for 0 < p < 2, (0, inf) for p >= 2
__device__ __forceinline__ bool glm_y_in_range(double p, double y) {
  const bool low = p <= 0.0 ? y > -INFINITY : (p < 2.0 ? y >= 0.0 : y > 0.0);
  return low && y < INFINITY;
}

// MODE kGlmGradient / kGlmHessian: per-CTA [loss, const, sum y, kept, y out of range, h <= 0, y not finite, 0 | g.x (d), sum g,
// zeros | (kGlmHessian) the Hessian blocks at kGlmHess, pitch kGlmHp]; kGlmLadder: the loss at step k in [k], k < n_steps.
// op: w [kMaxD], step [kMaxD], [b, db, negative label, positive label] (kGlmOp* in b2_internal.cuh).
// FAM kGlmTweedie: link and power select the loss.  kGlmBinomial: the half-binomial loss on the labels of op (link and
// power unused); sum y counts the positive rows, y out of range the rows with neither label, and slot 7 the rows
// classified correctly ((eta > 0) == positive label, a row with neither label never).  A compile-time family keeps the
// Tweedie instantiations as they were.
template <typename T, bool RING, int MODE, int FAM>
__global__ void __launch_bounds__(kTileThreads, 1)
glm_kernel(const T* __restrict__ X, int64_t n, int d, int64_t ldx, const float* __restrict__ y,
           const uint8_t* __restrict__ mask, int keep, const double* __restrict__ op, int link, double power,
           int n_steps, double* __restrict__ part) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  TileRing<T, RING, true> tiles{X, n, d, ldx, y, mask, keep, smem_u32(smem_raw)};
  const int dp = glm_dp(d), zp = tile_vpitch(dp), nb = dp / 16, nsb = nb * (nb + 1) / 2;
  double* Zs = reinterpret_cast<double*>(smem_raw + tile_ring_bytes(RING, true));   // [row][zp]: z = [x 1 0...]
  double* HZs = Zs + (MODE == kGlmHessian ? kTileRows * zp : 0);                   // |h| z
  double* wv = HZs + kTileRows * zp;       // [kMaxD] w
  double* sv = wv + kMaxD;                 // [kMaxD] the Newton step (kGlmLadder)
  double* yv = sv + kMaxD;                 // y (0 for rows not kept)
  double* gs = yv + kTileRows;             // g (0 for rows not kept)
  double* hs = gs + kTileRows;             // |h| (0 for rows not kept)
  double* red = hs + kTileRows;            // [warp][32] the warps' sums
  double* lsum = red + kTileWarps * 32;    // [warp][u][8] the scalar sums of the rows warp + 8 u (gradient / Hessian)
  double* gsum = lsum + kTileWarps * 32;   // [kMaxD + 8] the gradient sums, entry j of thread j
  int* sb = reinterpret_cast<int*>(gsum + kMaxD + 8);    // the upper blocks' table
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g8 = lane >> 2, t4 = lane & 3;
  for (int t = tid; t < kTileWarps * 32; t += blockDim.x) lsum[t] = 0.0;
  for (int t = tid; t < kMaxD + 8; t += blockDim.x) gsum[t] = 0.0;
  for (int t = tid; t < kMaxD; t += blockDim.x) {
    wv[t] = t < d ? op[kGlmOpW + t] : 0.0;
    sv[t] = (MODE == kGlmLadder && t < d) ? op[kGlmOpStep + t] : 0.0;
  }
  upper_blocks(sb, nb);
  const double b = op[kGlmOpMisc], db = op[kGlmOpMisc + 1];
  const int64_t n_tiles = (n + kTileRows - 1) / kTileRows;
  tiles.start();
  // kGlmLadder: lane k sums the loss at step k.  The other sums stay in shared memory (lsum, gsum), which leaves the
  // registers to the Hessian's accumulators.
  double s_loss = 0.0;
  double acc[kGlmSB][4][2] = {};
  if (!tiles.produce()) {
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
      // (1) the tile: z = [x 1 0...] and y, zero for rows not kept
      bool use[kTileRowsPerWarp];
      tiles.load(tile * kTileRows, dp, use,
                 [&](int r, int j, bool kept, bool live, float x) {
                   Zs[r * zp + j] = live ? (double)x : (kept && j == d ? 1.0 : 0.0);
                 },
                 [&](int r, bool, double yr) { yv[r] = yr; });
      __syncwarp();
      // (2) eta (and deta) of the warp's rows: every lane ends with the same value
      double eta[kTileRowsPerWarp], deta[kTileRowsPerWarp];
#pragma unroll
      for (int u = 0; u < kTileRowsPerWarp; ++u) {
        const double* zr = Zs + (warp + kTileWarps * u) * zp;
        double a = 0.0, c = 0.0;
        for (int j = lane; j < d; j += 32) {
          a = fma(zr[j], wv[j], a);
          if constexpr (MODE == kGlmLadder) c = fma(zr[j], sv[j], c);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          a += __shfl_xor_sync(0xffffffffu, a, o);
          if constexpr (MODE == kGlmLadder) c += __shfl_xor_sync(0xffffffffu, c, o);
        }
        eta[u] = a + b;
        deta[u] = c + db;
      }
      // (3) the pointwise terms
      if constexpr (MODE == kGlmLadder) {
        const double t = ldexp(1.0, -lane);           // t = 1, 1/2, ... 2^-20: lane k < n_steps takes step k
#pragma unroll
        for (int u = 0; u < kTileRowsPerWarp; ++u) {
          double l;
          if constexpr (FAM == kGlmBinomial)
            l = binom_ladder_loss(yv[warp + kTileWarps * u] == op[kGlmOpMisc + 3] ? 1.0 : 0.0, eta[u] + t * deta[u]);
          else
            l = glm_loss(link, power, yv[warp + kTileWarps * u], eta[u] + t * deta[u]);
          s_loss += (use[u] && lane < n_steps) ? l : 0.0;
        }
      } else {
        if (lane < kTileRowsPerWarp) {            // lane u takes row warp + 8 u
          double e = eta[0];
          bool kept = use[0];
#pragma unroll
          for (int u = 1; u < kTileRowsPerWarp; ++u) {
            e = lane == u ? eta[u] : e;
            kept = lane == u ? use[u] : kept;
          }
          const int r = warp + kTileWarps * lane;
          const double yy = yv[r];
          double l, gg, hh;
          double* ls = lsum + (warp * 4 + lane) * 8;
          if constexpr (FAM == kGlmBinomial) {
            const bool is_pos = yy == op[kGlmOpMisc + 3], in_range = is_pos || yy == op[kGlmOpMisc + 2];
            const double tt = is_pos ? 1.0 : 0.0;
            l = binom_loss(tt, e);
            binom_grad_hess(tt, e, gg, hh);
            ls[0] += kept ? l : 0.0;
            ls[2] += kept ? tt : 0.0;
            ls[3] += kept ? 1.0 : 0.0;
            ls[4] += (kept && !in_range) ? 1.0 : 0.0;
            ls[5] += (kept && hh <= 0.0) ? 1.0 : 0.0;
            ls[6] += (kept && !isfinite(yy)) ? 1.0 : 0.0;
            ls[kGlmCorrect] += (kept && in_range && (e > 0.0) == is_pos) ? 1.0 : 0.0;
          } else {
            glm_point(link, power, yy, e, l, gg, hh);
            const double cst = glm_const(link, power, yy);
            ls[0] += kept ? l : 0.0;
            ls[1] += kept ? cst : 0.0;
            ls[2] += kept ? yy : 0.0;
            ls[3] += kept ? 1.0 : 0.0;
            ls[4] += (kept && !glm_y_in_range(power, yy)) ? 1.0 : 0.0;
            ls[5] += (kept && hh <= 0.0) ? 1.0 : 0.0;
            ls[6] += (kept && !isfinite(yy)) ? 1.0 : 0.0;
          }
          gs[r] = kept ? gg : 0.0;
          hs[r] = kept ? fabs(hh) : 0.0;
        }
        tile_consumer_sync();
        // (4) the gradient, then (kGlmHessian) the |h|-scaled rows
        if (tid <= d) {
          double a = gsum[tid];
#pragma unroll 8
          for (int r = 0; r < kTileRows; ++r) a = fma(gs[r], Zs[r * zp + tid], a);
          gsum[tid] = a;
        }
        if constexpr (MODE == kGlmHessian) {
          for (int t = tid; t < kTileRows * dp; t += kTileConsumers) {
            const int r = t / dp, j = t - r * dp;
            HZs[r * zp + j] = hs[r] * Zs[r * zp + j];
          }
          tile_consumer_sync();
          // (5) H += (|h| z)^T z over the tile's rows, the warp's blocks
          upper_accumulate(acc, sb, nsb, [&](int r, int c) { return HZs[r * zp + c]; }, Zs, zp, warp, g8, t4);
        }
      }
      tile_consumer_sync();
    }
  }
  // the CTA's sums in a fixed order: the lanes of a warp, then the warps in order
  double* out = part + (size_t)blockIdx.x * kGlmPart;
  if constexpr (MODE == kGlmLadder) {
    if (warp < kTileWarps) red[warp * 32 + lane] = s_loss;
    __syncthreads();
    if (tid < 32) {
      double v = 0.0;
      for (int w = 0; w < kTileWarps; ++w) v += red[w * 32 + tid];
      out[tid] = v;
    }
  } else {
    __syncthreads();
    if (tid < kGlmHess) {                          // the scalars, the gradient, zeros in the unused entries
      double r = 0.0;
      if (tid < (FAM == kGlmBinomial ? kGlmCorrect + 1 : 7))
        for (int q = 0; q < kTileWarps * 4; ++q) r += lsum[q * 8 + tid];
      else if (tid >= kGlmGrad && tid <= kGlmGrad + d)
        r = gsum[tid - kGlmGrad];
      out[tid] = r;
    }
    if constexpr (MODE == kGlmHessian) upper_store(acc, sb, nsb, out + kGlmHess, kGlmHp, warp, g8, t4);
  }
}

// mu = exp(eta) (log link) or eta (identity) per row, eta = x.w + b in fp64: one warp per row
template <typename T>
__global__ void __launch_bounds__(256)
glm_predict_kernel(const T* __restrict__ X, int64_t n, int d, int64_t ldx, const double* __restrict__ op, int link,
                   double* __restrict__ mu) {
  __shared__ double wv[kMaxD];
  for (int t = threadIdx.x; t < kMaxD; t += blockDim.x) wv[t] = t < d ? op[kGlmOpW + t] : 0.0;
  __syncthreads();
  const double b = op[kGlmOpMisc];
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < n; row += warps) {
    const T* xr = X + row * ldx;
    double a = 0.0;
    for (int j = lane; j < d; j += 32) a = fma((double)ld_row_val<T>(xr + j), wv[j], a);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    if (lane == 0) mu[row] = link == B2_GLM_LOG ? exp(a + b) : a + b;
  }
}

// The logistic model's outputs per row, eta = x.w + b in fp64: one warp per row.  Each output may be null: eta; the
// probabilities [1 - p, p] with p = 1 / (1 + exp(-eta)) (scipy's expit, as sklearn's _predict_proba_lr computes it); the
// label, the positive one when eta > 0.
template <typename T>
__global__ void __launch_bounds__(256)
logistic_predict_kernel(const T* __restrict__ X, int64_t n, int d, int64_t ldx, const double* __restrict__ op,
                        double* __restrict__ decision, double* __restrict__ proba, float* __restrict__ label) {
  __shared__ double wv[kMaxD];
  for (int t = threadIdx.x; t < kMaxD; t += blockDim.x) wv[t] = t < d ? op[kGlmOpW + t] : 0.0;
  __syncthreads();
  const double b = op[kGlmOpMisc];
  const float neg = (float)op[kGlmOpMisc + 2], pos = (float)op[kGlmOpMisc + 3];
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); row < n; row += warps) {
    const T* xr = X + row * ldx;
    double a = 0.0;
    for (int j = lane; j < d; j += 32) a = fma((double)ld_row_val<T>(xr + j), wv[j], a);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    if (lane == 0) {
      const double eta = a + b;
      if (decision != nullptr) decision[row] = eta;
      if (proba != nullptr) {
        const double p = 1.0 / (1.0 + exp(-eta));
        proba[2 * row] = 1.0 - p;
        proba[2 * row + 1] = p;
      }
      if (label != nullptr) label[row] = eta > 0.0 ? pos : neg;
    }
  }
}

// The label scan of a device fp32 y over its kept rows (kLabel* in b2_internal.cuh): counts by integer atomics and the
// extremes by atomics on order-preserving keys (label_key, b2_internal.cuh), so the result does not depend on the order of
// the rows.
__device__ __forceinline__ unsigned long long warp_sum_u64(unsigned long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// pass 1: kept, not finite, finite but not integral, the smallest and largest key of the finite kept y
__global__ void __launch_bounds__(256)
label_scan_kernel(const float* __restrict__ y, int64_t n, const uint8_t* __restrict__ mask, int keep,
                  unsigned long long* __restrict__ st) {
  unsigned long long kept = 0, nonfinite = 0, nonint = 0, kmin = ~0ull, kmax = 0;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    if (mask != nullptr && __ldg(mask + i) != (uint8_t)keep) continue;
    const float v = __ldg(y + i);
    ++kept;
    if (!isfinite(v)) { ++nonfinite; continue; }
    nonint += v != rintf(v);
    const unsigned long long k = label_key(v);
    kmin = k < kmin ? k : kmin;
    kmax = k > kmax ? k : kmax;
  }
  kept = warp_sum_u64(kept);
  nonfinite = warp_sum_u64(nonfinite);
  nonint = warp_sum_u64(nonint);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long a = __shfl_xor_sync(0xffffffffu, kmin, o), c = __shfl_xor_sync(0xffffffffu, kmax, o);
    kmin = a < kmin ? a : kmin;
    kmax = c > kmax ? c : kmax;
  }
  if ((threadIdx.x & 31) == 0 && kept > 0) {
    atomicAdd(st + kLabelKept, kept);
    atomicAdd(st + kLabelNonFinite, nonfinite);
    atomicAdd(st + kLabelNonIntegral, nonint);
    atomicMin(st + kLabelMin, kmin);
    atomicMax(st + kLabelMax, kmax);
  }
}

// pass 2: the kept rows equal to the smallest and to the largest value
__global__ void __launch_bounds__(256)
label_count_kernel(const float* __restrict__ y, int64_t n, const uint8_t* __restrict__ mask, int keep,
                   unsigned long long* __restrict__ st) {
  if (st[kLabelMin] > st[kLabelMax]) return;            // no finite kept y
  const float lo = label_of_key(st[kLabelMin]), hi = label_of_key(st[kLabelMax]);
  unsigned long long n_lo = 0, n_hi = 0;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    if (mask != nullptr && __ldg(mask + i) != (uint8_t)keep) continue;
    const float v = __ldg(y + i);
    n_lo += v == lo;
    n_hi += v == hi;
  }
  n_lo = warp_sum_u64(n_lo);
  n_hi = warp_sum_u64(n_hi);
  if ((threadIdx.x & 31) == 0) {
    if (n_lo > 0) atomicAdd(st + kLabelNMin, n_lo);
    if (n_hi > 0) atomicAdd(st + kLabelNMax, n_hi);
  }
}

}  // namespace

// The rows [0, n) in the launches of scoring's plan: whole 32-row tiles of what plan_rows streams through the ring go to the
// ring flavour, the rest (or every row of another layout) to the direct one; each launch is followed by its ordered reduce
// into ctx->glm (`first_block` overwrites, otherwise adds).
int launch_glm(b2_ctx* ctx, const void* X, int x_dtype, int64_t n, int d, int64_t ldx, const float* y,
               const uint8_t* mask, int keep, int mode, int family, int link, double power, int n_steps,
               bool first_block) {
  return split_ring_rows(ctx, X, x_dtype, n, d, ldx, y, mask, kTileRows, first_block, [&](bool ring, const RowSpan& s) {
    // two CTAs per SM hide the latency of the per-tile steps where the shared memory allows it (all but the Hessian)
    const int grid = tile_grid(s.rows, ctx->sm_count, mode == kGlmHessian ? 1 : 2);
    const uint32_t smem = (uint32_t)glm_smem_bytes(glm_dp(d), ring, mode);
    const int rc = with_rows(x_dtype, s.X, [&](auto* Xr) {
      using T = row_t<decltype(Xr)>;
      return with_int<kGlmGradient, kGlmHessian, kGlmLadder>(mode, [&](auto M) {
        return with_int<kGlmTweedie, kGlmBinomial>(family, [&](auto F) {
          constexpr int MODE = decltype(M)::value, FAM = decltype(F)::value;
          auto kernel = ring ? glm_kernel<T, true, MODE, FAM> : glm_kernel<T, false, MODE, FAM>;
          return launch_smem(kernel, grid, tile_threads(ring), smem, ctx->stream, Xr, s.rows, d, ldx, s.y, s.mask,
                             keep, static_cast<const double*>(ctx->glm + kGlmOp), link, power, n_steps, ctx->glm_part);
        });
      });
    });
    if (rc != B2_OK) return rc;
    const int n_lin = mode == kGlmLadder ? 32 : kGlmHess, d1 = mode == kGlmHessian ? d + 1 : 0;
    return launch_ordered_reduce(ctx, ctx->glm_part, kGlmPart, grid, s.first, n_lin, 0u, ctx->glm, d1, kGlmHess, kGlmHp);
  });
}

int launch_glm_predict(b2_ctx* ctx, const void* X, int x_dtype, int64_t n, int d, int64_t ldx, int link, double* mu) {
  if (n == 0) return B2_OK;
  int64_t want = (n + 7) / 8;
  const int64_t cap = (int64_t)ctx->sm_count * 8;
  const int grid = (int)(want < cap ? want : cap);
  with_rows(x_dtype, X, [&](auto* Xr) {
    glm_predict_kernel<<<grid, 256, 0, ctx->stream>>>(Xr, n, d, ldx, ctx->glm + kGlmOp, link, mu);
    return B2_OK;
  });
  B2_CUDA(cudaGetLastError());
  ctx->launches += 1;
  return B2_OK;
}

int launch_logistic_predict(b2_ctx* ctx, const void* X, int x_dtype, int64_t n, int d, int64_t ldx, double* decision,
                            double* proba, float* label) {
  if (n == 0) return B2_OK;
  const int64_t want = (n + 7) / 8, cap = (int64_t)ctx->sm_count * 8;
  const int grid = (int)(want < cap ? want : cap);
  with_rows(x_dtype, X, [&](auto* Xr) {
    logistic_predict_kernel<<<grid, 256, 0, ctx->stream>>>(Xr, n, d, ldx, ctx->glm + kGlmOp, decision, proba, label);
    return B2_OK;
  });
  B2_CUDA(cudaGetLastError());
  ctx->launches += 1;
  return B2_OK;
}

int launch_label_scan(b2_ctx* ctx, const float* y, int64_t n, const uint8_t* mask, int keep, unsigned long long* st) {
  B2_CUDA(cudaMemsetAsync(st, 0, sizeof(unsigned long long) * kLabelWords, ctx->stream));
  B2_CUDA(cudaMemsetAsync(st + kLabelMin, 0xff, sizeof(unsigned long long), ctx->stream));
  if (n == 0) return B2_OK;
  const int64_t want = (n + 2047) / 2048, cap = (int64_t)ctx->sm_count * 8;
  const int grid = (int)(want < cap ? want : cap);
  label_scan_kernel<<<grid, 256, 0, ctx->stream>>>(y, n, mask, keep, st);
  B2_CUDA(cudaGetLastError());
  label_count_kernel<<<grid, 256, 0, ctx->stream>>>(y, n, mask, keep, st);
  B2_CUDA(cudaGetLastError());
  ctx->launches += 2;
  return B2_OK;
}

}  // namespace b2
