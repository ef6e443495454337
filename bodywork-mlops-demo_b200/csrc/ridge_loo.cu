// ridge_loo.cu -- the leave-one-out pass of RidgeCV(alphas).fit(X, y) with cv=None (b2_ridge_loo; DESIGN.md section 6),
// and its T-target form for RidgeClassifierCV (b2_ridge_classifier_loo; section 13, at the end of this file).
//
// With A = Q diag(lambda) Q^T the centred Gram of the kept rows, c = Q^T r and w_ja = 1 / (lambda_j + alpha_a), a kept
// row's leave-one-out error at alpha_a is e = ((y - ybar) - yhat) / (1 - h) with z = Q^T (x - m), yhat = sum_j z_j c_j
// w_ja and h = h0 + sum_j z_j^2 w_ja: what scikit-learn's _RidgeGCV computes from an SVD of the whole design matrix.  Per
// row that is 2 D^2 + 4 A D flops against D * 4 bytes of row: the pass is fp64-compute bound, so both products run on the
// fp64 tensor core (mma.sync m8n8k4 f64):
//   (1) a tile of 32 rows -> shared memory as v = x - m in fp64 from the stored value (one rounding), 0 for rows not kept;
//   (2) Z = V Q (Q resident in shared memory for the whole launch), written back over V;
//   (3) [yhat | h - h0] = [Z (c o w) | (Z o Z) w], the B operands read from a D x 64 table built once per call; the
//       per-row, per-alpha epilogue forms e in fp64 (y - yhat cancels) and adds e^2 to the lane's sums.
// The rows take scoring's plan (plan_rows): where it streams contiguous rows through the bulk-copy ring, a producer warp
// runs ring_produce with 32-row tiles of X and y and the consumers convert each slot in (1); the rows after the last whole
// tile, and every other layout, are read by the same consumers straight from global memory.
// A row not kept has v = 0 and e = 0 by selects, so whatever it holds never reaches a sum.  Each CTA writes its sums per
// alpha in a fixed order; the ordered reduce adds the CTAs in order, so two calls return identical sums.
#include "b2_internal.cuh"
#include "b2_dmma.cuh"

namespace b2 {
namespace {

size_t loo_smem_bytes(int dp, bool ring) {
  return tile_ring_bytes(ring, true) +
         sizeof(double) * ((size_t)dp * tile_bpitch(dp) + (size_t)kTileRows * tile_vpitch(dp) + 2 * kTileRows + kMaxD +
                           (size_t)kTileWarps * kMaxAlphas);
}

// the B operands of (3): Cw[j][a] = c_j / (lambda_j + alpha_a), W[j][a] = 1 / (lambda_j + alpha_a); 0 outside d x n_alphas
__global__ void loo_prep_kernel(double* __restrict__ loo, int d, int n_alphas) {
  for (int t = threadIdx.x; t < kMaxD * kMaxAlphas; t += blockDim.x) {
    const int j = t / kMaxAlphas, a = t - j * kMaxAlphas;
    double cw = 0.0, w = 0.0;
    if (j < d && a < n_alphas) {
      w = 1.0 / (loo[kLooLam + j] + loo[kLooAlpha + a]);
      cw = loo[kLooC + j] * w;
    }
    loo[kLooCw + t] = cw;
    loo[kLooW + t] = w;
  }
}

// RING: rows [0, n), n a multiple of kTileRows, contiguous (ldx == d) and 16-byte aligned with y, through the bulk-copy
// ring; otherwise rows [0, n) of any layout (stride ldx, fp32 or bf16, any alignment) from global memory.  Tiles
// blockIdx.x, + gridDim.x, ...
// Work of (3): the n_alphas are ceil(n_alphas / 8) n-tiles; each gets G = 8 / n-tiles warps, each warp a group of
// ceil(kTileMT / G) m-tiles, so every warp holds at most one (n-tile, group) for the whole launch and its sums stay in
// registers.
template <typename T, bool RING>
__global__ void __launch_bounds__(kTileThreads, 1)
loo_kernel(const T* __restrict__ X, int64_t n, int d, int64_t ldx, const float* __restrict__ y,
           const uint8_t* __restrict__ mask, int keep, const double* __restrict__ loo, int n_alphas,
           double* __restrict__ cv, double* __restrict__ part) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  TileRing<T, RING, true> tiles{X, n, d, ldx, y, mask, keep, smem_u32(smem_raw)};
  const int dp = tile_dp(d), qp = tile_bpitch(dp), vp = tile_vpitch(dp);
  double* Qs = reinterpret_cast<double*>(smem_raw + tile_ring_bytes(RING, true));   // Q[i][k], zero padded to dp x dp
  double* Vs = Qs + dp * qp;               // the tile: v = x - m, then Z = V Q
  double* yc = Vs + kTileRows * vp;        // y - ybar (0 for rows not kept)
  double* usef = yc + kTileRows;           // 1: kept
  double* mean = usef + kTileRows;         // [kMaxD]
  double* sums = mean + kMaxD;             // [group][kMaxAlphas]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t4 = lane & 3;
  for (int t = tid; t < dp * dp; t += blockDim.x) {
    const int i = t / dp, k = t - i * dp;
    Qs[i * qp + k] = (i < d && k < d) ? loo[kLooQ + i * kMaxD + k] : 0.0;
  }
  for (int t = tid; t < kMaxD; t += blockDim.x) mean[t] = t < d ? loo[kLooMean + t] : 0.0;
  for (int t = tid; t < kTileWarps * kMaxAlphas; t += blockDim.x) sums[t] = 0.0;
  const double ybar = loo[kLooMisc], h0 = loo[kLooMisc + 2];
  const int na = (n_alphas + 7) >> 3;
  const int G = kTileWarps / na, mpg = (kTileMT + G - 1) / G;
  const bool has_item = warp < na * G;     // warp-uniform
  const int nt_a = has_item ? warp / G : 0, grp = has_item ? warp % G : 0, mt0 = grp * mpg;
  const int a0 = 8 * nt_a + 2 * t4;        // the two alphas of this lane's accumulators
  const int ab = 8 * nt_a + g;             // the alpha of this lane's B fragment
  const int64_t n_tiles = (n + kTileRows - 1) / kTileRows;
  tiles.start();
  if (!tiles.produce()) {
    double acc_e[2] = {0.0, 0.0};
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
      const int64_t row0 = tile * kTileRows;
      // (1) the tile: v = x - m, y - ybar and 1 for kept rows, 0 for the others
      tiles.load(row0, dp,
                 [&](int r, int j, bool, bool live, float x) { Vs[r * vp + j] = live ? (double)x - mean[j] : 0.0; },
                 [&](int r, bool kept, double yr) {
                   yc[r] = kept ? yr - ybar : 0.0;
                   usef[r] = kept ? 1.0 : 0.0;
                 });
      tile_consumer_sync();
      // (2) Z = V Q: warp w takes the n-tiles w and w + 8 of the dp / 8, all m-tiles
      double z[2][kTileMT][2];
      tile_product(Vs, vp, Qs, qp, dp, dp / 8, z);
      tile_consumer_sync();
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int nt = warp + kTileWarps * u;
        if (nt < dp / 8) {
#pragma unroll
          for (int mt = 0; mt < kTileMT; ++mt) {
            Vs[(8 * mt + g) * vp + 8 * nt + 2 * t4] = z[u][mt][0];
            Vs[(8 * mt + g) * vp + 8 * nt + 2 * t4 + 1] = z[u][mt][1];
          }
        }
      }
      tile_consumer_sync();
      // (3) yhat and h of every kept row and alpha, then e^2
      if (has_item) {
        double yh[kTileMT][2], hh[kTileMT][2];
#pragma unroll
        for (int mm = 0; mm < kTileMT; ++mm) { yh[mm][0] = yh[mm][1] = hh[mm][0] = hh[mm][1] = 0.0; }
        for (int ks = 0; ks < dp / 4; ++ks) {
          const int j = 4 * ks + t4;
          const double bc = __ldg(loo + kLooCw + j * kMaxAlphas + ab);
          const double bw = __ldg(loo + kLooW + j * kMaxAlphas + ab);
#pragma unroll
          for (int mm = 0; mm < kTileMT; ++mm) {
            if (mm < mpg && mt0 + mm < kTileMT) {              // warp-uniform
              const double zz = Vs[(8 * (mt0 + mm) + g) * vp + j];
              dmma(yh[mm][0], yh[mm][1], zz, bc);
              dmma(hh[mm][0], hh[mm][1], zz * zz, bw);
            }
          }
        }
#pragma unroll
        for (int mm = 0; mm < kTileMT; ++mm) {
          if (mm < mpg && mt0 + mm < kTileMT) {
            const int r = 8 * (mt0 + mm) + g;
            const int64_t row = row0 + r;
            const bool kept = usef[r] != 0.0;
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const double err = kept ? (yc[r] - yh[mm][e]) / (1.0 - (h0 + hh[mm][e])) : 0.0;
              const double e2 = err * err;
              acc_e[e] += e2;
              const int a = a0 + e;
              if (cv != nullptr && row < n && a < n_alphas)
                cv[row * n_alphas + a] = kept ? e2 : __longlong_as_double(0x7ff8000000000000ll);
            }
          }
        }
      }
      tile_consumer_sync();
    }
    // the CTA's sums: the 8 row lanes of an alpha pair combined, then the groups of an alpha in group order
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      double v = acc_e[e];
#pragma unroll
      for (int o = 4; o < 32; o <<= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (has_item && g == 0) sums[grp * kMaxAlphas + a0 + e] = v;
    }
  }
  __syncthreads();
  for (int a = tid; a < kMaxAlphas; a += blockDim.x) {
    double v = 0.0;
    for (int q = 0; q < kTileWarps; ++q) v += sums[q * kMaxAlphas + a];
    part[(size_t)blockIdx.x * kMaxAlphas + a] = v;
  }
}

// ---- RidgeClassifierCV (b2_ridge_classifier_loo; DESIGN.md section 13) ------------------------------------------------
// The same error with T targets t_k = +1 where the row's class is k (class 1 when T = 1), -1 otherwise, centred by
// ybar_k = 2 n_k / n - 1: per kept row and alpha, h is shared and yhat_k = sum_j z_j C_jk w_ja with C = Q^T R, R the
// class-sum right-hand sides 2 (s_k - (n_k / n) s) of solve_classes_kernel.  Per 32-row tile: (1) and (2) as loo_kernel,
// (3) h - h0 = (Z o Z) w, then per target k the 8-alpha column chunk yhat_k = Z (C_k o w) and its epilogue: e_k =
// ((t_k - ybar_k) - yhat_k) / (1 - h) adds e_k^2 to the alpha's sum and p_k = t_k - e_k to the row's running first
// argmax.  The T A prediction columns are never in shared memory together; one read of the rows serves every alpha.

// The B operands: W[j][a] = 1 / (lambda_j + alpha_a), C = Q^T R and CW[j][k 8 ceil(A / 8) + a] = C_jk W[j][a], 0 outside
// d x n_alphas (rows up to the padded dp), and ybar.  One CTA.
constexpr int kLcPrepThreads = 1024;
__global__ void __launch_bounds__(kLcPrepThreads)
loo_classes_prep_kernel(const double* __restrict__ loo, const double* __restrict__ cls, int d, int n_classes,
                        int n_alphas, int fit_intercept, double* __restrict__ lc) {
  __shared__ double R[kMaxD * kMaxClasses];          // R[i][k], pitch kMaxClasses
  __shared__ double tot[kMaxD];
  const int tid = threadIdx.x, T = n_classes == 2 ? 1 : n_classes, dp = tile_dp(d);
  const int ap = 8 * ((n_alphas + 7) / 8), cwp = T * ap;
  const double* sums = cls + kClsSums;               // [K][d + 1]
  const double n = loo[kLooMisc + 1];
  if (tid < d) {
    double s = 0.0;
    for (int k = 0; k < n_classes; ++k) s += sums[k * (d + 1) + tid];
    tot[tid] = s;
  }
  __syncthreads();
  for (int t = tid; t < T * d; t += blockDim.x) {
    const int tt = t / d, i = t - tt * d, k = T == 1 ? 1 : tt;
    const double sk = sums[k * (d + 1) + i], nk = sums[k * (d + 1) + d];
    R[i * kMaxClasses + tt] = fit_intercept ? 2.0 * (sk - (nk / n) * tot[i]) : 2.0 * sk - tot[i];
  }
  if (tid < T) {
    const int k = T == 1 ? 1 : tid;
    lc[kLcYbar + tid] = fit_intercept ? 2.0 * sums[k * (d + 1) + d] / n - 1.0 : 0.0;
  }
  __syncthreads();
  for (int t = tid; t < d * T; t += blockDim.x) {
    const int j = t / T, k = t - j * T;
    double c = 0.0;
    for (int i = 0; i < d; ++i) c = fma(loo[kLooQ + i * kMaxD + j], R[i * kMaxClasses + k], c);
    lc[kLcC + j * kMaxClasses + k] = c;
  }
  for (int t = tid; t < kMaxD * kMaxAlphas; t += blockDim.x) {
    const int j = t / kMaxAlphas, a = t - j * kMaxAlphas;
    lc[kLcW + t] = (j < d && a < n_alphas) ? 1.0 / (loo[kLooLam + j] + loo[kLooAlpha + a]) : 0.0;
  }
  __syncthreads();                                   // C and W, written above by other threads of the CTA
  for (int t = tid; t < dp * cwp; t += blockDim.x) {
    const int j = t / cwp, c = t - j * cwp, k = c / ap, a = c - k * ap;
    lc[kLcCw + t] = (j < d && a < n_alphas) ? lc[kLcC + j * kMaxClasses + k] * lc[kLcW + j * kMaxAlphas + a] : 0.0;
  }
}

// the tile region: the tile [kTileRows][vp], after the last tile the CTA's sums [kTileWarps][kLcPart]
__host__ __device__ inline int loo_classes_tile_doubles(int vp) {
  return kTileRows * vp > kTileWarps * kLcPart ? kTileRows * vp : kTileWarps * kLcPart;
}
size_t loo_classes_smem_bytes(int dp, bool ring) {
  return tile_ring_bytes(ring, true) +
         sizeof(double) * ((size_t)dp * tile_bpitch(dp) + loo_classes_tile_doubles(tile_vpitch(dp)) + kMaxD +
                           kMaxClasses) +
         sizeof(float) * kMaxClasses + sizeof(int) * kTileRows;
}

// Rows and warps as loo_kernel: each warp holds one (8-alpha n-tile, group of m-tiles) for the whole launch and runs
// its T prediction chunks one after the other.  Per CTA: part[a] = sum e^2 over its kept rows and every target,
// part[kMaxAlphas + a] = its kept rows whose first argmax of p is their class (every kept row when T = 1).  cv (not
// null): [row][T][n_alphas] e^2, or p with `accuracy`; NaN for rows not kept.
template <typename T, bool RING>
__global__ void __launch_bounds__(kTileThreads, 1)
loo_classes_kernel(const T* __restrict__ X, int64_t n, int d, int64_t ldx, const float* __restrict__ y,
                   const uint8_t* __restrict__ mask, int keep, const double* __restrict__ loo,
                   const double* __restrict__ cls_op, const double* __restrict__ lc, int n_classes, int n_alphas,
                   int accuracy, double* __restrict__ cv, double* __restrict__ part) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  TileRing<T, RING, true> tiles{X, n, d, ldx, y, mask, keep, smem_u32(smem_raw)};
  const int dp = tile_dp(d), qp = tile_bpitch(dp), vp = tile_vpitch(dp), nT = n_classes == 2 ? 1 : n_classes;
  double* Qs = reinterpret_cast<double*>(smem_raw + tile_ring_bytes(RING, true));   // Q[i][k], zero padded to dp x dp
  double* Vs = Qs + dp * qp;               // the tile: v = x - m, then Z = V Q; the CTA's sums after the last tile
  double* mean = Vs + loo_classes_tile_doubles(vp);   // [kMaxD]
  double* ybar = mean + kMaxD;             // [kMaxClasses]
  float* cls = reinterpret_cast<float*>(ybar + kMaxClasses);
  int* row_class = reinterpret_cast<int*>(cls + kMaxClasses);   // the row's class, -1: none, -2: not kept
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t4 = lane & 3;
  for (int t = tid; t < dp * dp; t += blockDim.x) {
    const int i = t / dp, k = t - i * dp;
    Qs[i * qp + k] = (i < d && k < d) ? loo[kLooQ + i * kMaxD + k] : 0.0;
  }
  for (int t = tid; t < kMaxD; t += blockDim.x) mean[t] = t < d ? loo[kLooMean + t] : 0.0;
  for (int t = tid; t < kMaxClasses; t += blockDim.x) {
    ybar[t] = t < nT ? lc[kLcYbar + t] : 0.0;
    cls[t] = t < n_classes ? (float)cls_op[kClsClasses + t] : 0.f;
  }
  const double h0 = loo[kLooMisc + 2];
  const int na = (n_alphas + 7) >> 3, cwp = nT * 8 * na;
  const int G = kTileWarps / na, mpg = (kTileMT + G - 1) / G;
  const bool has_item = warp < na * G;     // warp-uniform
  const int nt_a = has_item ? warp / G : 0, grp = has_item ? warp % G : 0, mt0 = grp * mpg;
  const int a0 = 8 * nt_a + 2 * t4;        // the two alphas of this lane's accumulators
  const int ab = 8 * nt_a + g;             // the alpha of this lane's B fragment
  const int64_t n_tiles = (n + kTileRows - 1) / kTileRows;
  tiles.start();
  if (!tiles.produce()) {
    double acc_e[2] = {0.0, 0.0}, acc_c[2] = {0.0, 0.0};
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
      const int64_t row0 = tile * kTileRows;
      // (1) the tile: v = x - m, and each row's class
      tiles.load(row0, dp,
                 [&](int r, int j, bool, bool live, float x) { Vs[r * vp + j] = live ? (double)x - mean[j] : 0.0; },
                 [&](int r, bool kept, double yr) { row_class[r] = kept ? class_of(cls, n_classes, (float)yr) : -2; });
      tile_consumer_sync();
      // (2) Z = V Q
      double z[2][kTileMT][2];
      tile_product(Vs, vp, Qs, qp, dp, dp / 8, z);
      tile_consumer_sync();
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int nt = warp + kTileWarps * u;
        if (nt < dp / 8) {
#pragma unroll
          for (int mt = 0; mt < kTileMT; ++mt) {
            Vs[(8 * mt + g) * vp + 8 * nt + 2 * t4] = z[u][mt][0];
            Vs[(8 * mt + g) * vp + 8 * nt + 2 * t4 + 1] = z[u][mt][1];
          }
        }
      }
      tile_consumer_sync();
      if (has_item) {
        // (3) 1 / (1 - h) of the warp's rows and alphas
        double hinv[kTileMT][2];
#pragma unroll
        for (int mm = 0; mm < kTileMT; ++mm) { hinv[mm][0] = hinv[mm][1] = 0.0; }
#pragma unroll 8
        for (int ks = 0; ks < dp / 4; ++ks) {
          const int j = 4 * ks + t4;
          const double bw = __ldg(lc + kLcW + j * kMaxAlphas + ab);
#pragma unroll
          for (int mm = 0; mm < kTileMT; ++mm) {
            if (mm < mpg && mt0 + mm < kTileMT) {              // warp-uniform
              const double zz = Vs[(8 * (mt0 + mm) + g) * vp + j];
              dmma(hinv[mm][0], hinv[mm][1], zz * zz, bw);
            }
          }
        }
#pragma unroll
        for (int mm = 0; mm < kTileMT; ++mm) {
          hinv[mm][0] = 1.0 / (1.0 - (h0 + hinv[mm][0]));
          hinv[mm][1] = 1.0 / (1.0 - (h0 + hinv[mm][1]));
        }
        // per target: the chunk yhat_k, e_k, and the running first argmax of p
        double best[kTileMT][2];
        int best_k[kTileMT][2];
        for (int k = 0; k < nT; ++k) {
          double yh[kTileMT][2];
#pragma unroll
          for (int mm = 0; mm < kTileMT; ++mm) { yh[mm][0] = yh[mm][1] = 0.0; }
#pragma unroll 8                             // the B loads of 8 k-steps in flight ahead of their DMMAs
          for (int ks = 0; ks < dp / 4; ++ks) {
            const int j = 4 * ks + t4;
            const double bc = __ldg(lc + kLcCw + j * cwp + 8 * na * k + ab);
#pragma unroll
            for (int mm = 0; mm < kTileMT; ++mm) {
              if (mm < mpg && mt0 + mm < kTileMT) {
                const double zz = Vs[(8 * (mt0 + mm) + g) * vp + j];
                dmma(yh[mm][0], yh[mm][1], zz, bc);
              }
            }
          }
          const int target_class = nT == 1 ? 1 : k;
#pragma unroll
          for (int mm = 0; mm < kTileMT; ++mm) {
            if (mm < mpg && mt0 + mm < kTileMT) {
              const int r = 8 * (mt0 + mm) + g;
              const int64_t row = row0 + r;
              const int rc = row_class[r];
              const bool kept = rc != -2;
              const double tk = rc == target_class ? 1.0 : -1.0;
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const double err = kept ? ((tk - ybar[k]) - yh[mm][e]) * hinv[mm][e] : 0.0;
                const double p = tk - err;
                acc_e[e] += err * err;
                if (k == 0 || p > best[mm][e]) { best[mm][e] = p; best_k[mm][e] = k; }
                const int a = a0 + e;
                if (cv != nullptr && row < n && a < n_alphas)
                  cv[(row * nT + k) * n_alphas + a] =
                      kept ? (accuracy ? p : err * err) : __longlong_as_double(0x7ff8000000000000ll);
              }
            }
          }
        }
        // a kept row is right where the first argmax of p is the first argmax of t: its class (0 for no class)
#pragma unroll
        for (int mm = 0; mm < kTileMT; ++mm) {
          if (mm < mpg && mt0 + mm < kTileMT) {
            const int rc = row_class[8 * (mt0 + mm) + g];
            const int want = rc >= 0 ? rc : 0;
#pragma unroll
            for (int e = 0; e < 2; ++e) acc_c[e] += (rc != -2 && (nT == 1 || best_k[mm][e] == want)) ? 1.0 : 0.0;
          }
        }
      }
      tile_consumer_sync();
    }
    // the CTA's sums in the tile region: the 8 row lanes of an alpha pair combined, then the groups in group order
    double* sums = Vs;                       // [group][kLcPart]
    for (int t = tid; t < kTileWarps * kLcPart; t += kTileConsumers) sums[t] = 0.0;
    tile_consumer_sync();
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      double ve = acc_e[e], vc = acc_c[e];
#pragma unroll
      for (int o = 4; o < 32; o <<= 1) {
        ve += __shfl_xor_sync(0xffffffffu, ve, o);
        vc += __shfl_xor_sync(0xffffffffu, vc, o);
      }
      if (has_item && g == 0) {
        sums[grp * kLcPart + a0 + e] = ve;
        sums[grp * kLcPart + kMaxAlphas + a0 + e] = vc;
      }
    }
  }
  __syncthreads();
  for (int a = tid; a < kLcPart; a += blockDim.x) {
    double v = 0.0;
    for (int q = 0; q < kTileWarps; ++q) v += Vs[q * kLcPart + a];
    part[(size_t)blockIdx.x * kLcPart + a] = v;
  }
}

}  // namespace

// The rows [0, n) in the launches of scoring's plan: whole 32-row tiles of what plan_rows streams through the ring go to the
// ring flavour, the rest (or every row of another layout) to the direct one; each launch is followed by its ordered reduce.
int launch_loo(b2_ctx* ctx, const void* X, int x_dtype, int64_t n, int d, int64_t ldx, const float* y,
               const uint8_t* mask, int keep, int n_alphas, double* cv, bool first_block) {
  if (first_block) {
    loo_prep_kernel<<<1, 256, 0, ctx->stream>>>(ctx->loo, d, n_alphas);
    B2_CUDA(cudaGetLastError());
    ctx->launches += 1;
  }
  return split_ring_rows(ctx, X, x_dtype, n, d, ldx, y, mask, kTileRows, first_block, [&](bool ring, const RowSpan& s) {
    const int grid = tile_grid(s.rows, ctx->sm_count, 1);
    double* cvt = cv != nullptr ? cv + s.r0 * n_alphas : nullptr;
    const uint32_t smem = (uint32_t)loo_smem_bytes(tile_dp(d), ring);
    const int rc = with_rows(x_dtype, s.X, [&](auto* Xr) {
      using T = row_t<decltype(Xr)>;
      auto kernel = ring ? loo_kernel<T, true> : loo_kernel<T, false>;
      return launch_smem(kernel, grid, tile_threads(ring), smem, ctx->stream, Xr, s.rows, d, ldx, s.y, s.mask, keep,
                         static_cast<const double*>(ctx->loo), n_alphas, cvt, ctx->loo_part);
    });
    if (rc != B2_OK) return rc;
    return launch_ordered_reduce(ctx, ctx->loo_part, kMaxAlphas, grid, s.first, kMaxAlphas, 0u, ctx->loo + kLooSum);
  });
}

int launch_loo_classes(b2_ctx* ctx, const void* X, int x_dtype, int64_t n, int d, int64_t ldx, const float* y,
                       const uint8_t* mask, int keep, int n_classes, int n_alphas, int fit_intercept, bool accuracy,
                       double* cv, bool first_block) {
  if (first_block) {
    loo_classes_prep_kernel<<<1, kLcPrepThreads, 0, ctx->stream>>>(ctx->loo, ctx->cls, d, n_classes, n_alphas,
                                                                   fit_intercept, ctx->loo_cls);
    B2_CUDA(cudaGetLastError());
    ctx->launches += 1;
  }
  const int n_targets = n_classes == 2 ? 1 : n_classes;
  return split_ring_rows(ctx, X, x_dtype, n, d, ldx, y, mask, kTileRows, first_block, [&](bool ring, const RowSpan& s) {
    const int grid = tile_grid(s.rows, ctx->sm_count, 1);
    double* cvt = cv != nullptr ? cv + s.r0 * n_targets * n_alphas : nullptr;
    const uint32_t smem = (uint32_t)loo_classes_smem_bytes(tile_dp(d), ring);
    const int rc = with_rows(x_dtype, s.X, [&](auto* Xr) {
      using T = row_t<decltype(Xr)>;
      auto kernel = ring ? loo_classes_kernel<T, true> : loo_classes_kernel<T, false>;
      return launch_smem(kernel, grid, tile_threads(ring), smem, ctx->stream, Xr, s.rows, d, ldx, s.y, s.mask, keep,
                         static_cast<const double*>(ctx->loo), static_cast<const double*>(ctx->cls),
                         static_cast<const double*>(ctx->loo_cls), n_classes, n_alphas, accuracy ? 1 : 0, cvt,
                         ctx->glm_part);
    });
    if (rc != B2_OK) return rc;
    return launch_ordered_reduce(ctx, ctx->glm_part, kLcPart, grid, s.first, kLcPart, 0u, ctx->loo_cls + kLcSum);
  });
}

}  // namespace b2
