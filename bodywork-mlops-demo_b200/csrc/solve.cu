// solve.cu -- single-SM fp64 solve of the centred (ridge) normal equations from S.
//
// Replaces scipy.linalg.lstsq + _set_intercept inside LinearRegression.fit
// (stage_1_train_model.py:105-106 -> sklearn/linear_model/_base.py: `linalg.lstsq(Xc, yc, cond=tol)`
// then `intercept_ = y_offset - X_offset @ coef_`).  Ridge term as sklearn/linear_model/_ridge.py
// (`(Xc^T Xc + alpha I) w = Xc^T yc`).
//
//   solve_cholesky_kernel : A = Xc^T Xc + alpha I = L L^T in shared memory, two triangular solves.
//   solve_spectral_kernel : one-sided Jacobi on A (A V = W, columns of W orthogonal => w_k = lambda_k v_k):
//                           singular_ = sqrt(max(lambda, 0)) (descending), rank_ = #{singular > cond * max},
//                           coef = minimum-norm solution = what gelsd returns for rank-deficient X.
//
// One CTA: the matrices are <= 128 x 128 fp64 (132 KB with padding) -- latency bound, not a
// throughput problem (D^3/3 = 0.7 MFLOP).
#include "b2_internal.cuh"
#include "b2_xchg.cuh"

namespace b2 {
namespace {

constexpr int kOutIntercept = kMaxD;      // solve_out layout: [0,d) coef | intercept | info | rank | singular[d]
constexpr int kOutInfo = kMaxD + 1;
constexpr int kOutRank = kMaxD + 2;
constexpr int kOutSingular = kMaxD + 3;
constexpr int kOutRows = kOutSingular + kMaxD;   // eigvals kernel only

// Element i of a statistic (pitch d + 2) read through L2 (__ldcg: the fused solve has just written S from this CTA).
struct LdcgStat {
  const double* S;
  __device__ __forceinline__ double operator()(int i) const { return __ldcg(S + i); }
};

// Builds A (pitch d+1) and r in shared memory from the raw statistic `S` (S(i) = element i); returns means.  The loads
// of a whole batch are issued before the first use -- the phase is two L2 round trips, not one per element.
template <class Stat>
__device__ void build_normal_equations_of(const Stat& S, int d, double alpha, int fit_intercept,
                                       double* A, double* r, double* mean, double* ybar_out) {
  const int dp = d + 2, pitch = d + 1;
  const double n = S(d * dp + d);
  const double inv_n = n > 0.0 ? 1.0 / n : 0.0;
  double sxy = 0.0;
  if ((int)threadIdx.x < d) {
    const double sx = S(threadIdx.x * dp + d);
    sxy = S(threadIdx.x * dp + d + 1);
    mean[threadIdx.x] = fit_intercept ? sx * inv_n : 0.0;
  }
  const double ybar = fit_intercept ? S(d * dp + d + 1) * inv_n : 0.0;
  __syncthreads();
  if ((int)threadIdx.x < d) r[threadIdx.x] = sxy - n * mean[threadIdx.x] * ybar;
  // S is symmetric by construction (tc_fold / the SIMT reduce write both halves).  One warp per row, lane = column
  // (+32 u): no index division; two rows = 8 loads are issued before the first use.
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  for (int i0 = warp; i0 < d; i0 += 2 * nwarps) {
    const int i1 = i0 + nwarps;
    double v[8];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int j = lane + 32 * u;
      v[u] = j < d ? S(i0 * dp + j) : 0.0;
      v[4 + u] = (j < d && i1 < d) ? S(i1 * dp + j) : 0.0;
    }
    const double m0 = mean[i0], m1 = i1 < d ? mean[i1] : 0.0;
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int j = lane + 32 * u;
      if (j < d) {
        const double mj = mean[j];
        A[i0 * pitch + j] = v[u] - n * m0 * mj + (i0 == j ? alpha : 0.0);
        if (i1 < d) A[i1 * pitch + j] = v[4 + u] - n * m1 * mj + (i1 == j ? alpha : 0.0);
      }
    }
  }
  if (threadIdx.x == 0) *ybar_out = ybar;
  __syncthreads();
}

__device__ __forceinline__ void build_normal_equations(const double* S, int d, double alpha, int fit_intercept,
                                                       double* A, double* r, double* mean, double* ybar_out) {
  build_normal_equations_of(LdcgStat{S}, d, alpha, fit_intercept, A, r, mean, ybar_out);
}

// 1/x for positive x without the library division (a dependent `1.0 / x` is a long call sequence, several times the
// latency of a few dependent fp64 FMAs): the fp64 MUFU seed
// (rcp.approx.ftz.f64, ~2^-20 relative) and one cubic step y = y0 (1 + e + e^2), e = 1 - x y0 -- error e^3, below the
// rounding of the last FMA.  MUFU + 3 dependent FMAs; the pivot recurrence of the factorisation is paced by this chain.
__device__ __forceinline__ double rcp_pos(double x) {
  double y;
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(x));
  const double er = fma(-x, y, 1.0);
  const double t = fma(er, er, er);
  return fma(y, t, y);
}

// Peer exchange consumed by the solve (fused fit, b2_fit): wait for the exchange, sum the slots into S.
struct SolveXchg {
  double* own;                  // nullptr: S is already complete
  int n_ranks;
  unsigned int epoch;
  unsigned long long timeout_ns;
};

// Blocked right-looking LDL^T (block 16, no square roots) of the augmented matrix [A ; r^T]:  A = M D M^T with M unit
// lower triangular.  Carrying r as one extra row through the panel / update steps leaves w = D^-1 M^-1 r in that row, so
// there is no forward substitution; the back substitution M^T b = w needs no division.  fp64 arithmetic here is
// latency bound (the whole solve is 0.7 MFLOP), so every phase is written to keep the dependent chains short:
//   (1) diagonal block: one warp, 16 rows x 2 column halves in registers, pivots by shuffle; the products u_ik u_ck are
//       formed before the reciprocal of the pivot arrives, so the recurrence pivot -> next pivot is shuffle + rcp_pos +
//       one FMA, and a lane issues at most 8 column updates per pivot (the phase is issue bound on its one warp);
//   (2) panel: 4 lanes per row (the owner of column m broadcasts it inside the quad): shuffle + multiply + FMA per column;
//   (3) trailing update A[i][j] -= sum_m M[i][m] U[j][m] (U = M D, the unscaled entries) as 8 x 8 tiles on the fp64
//       tensor-core path (DMMA m8n8k4), 4 per tile, tiles of the lower triangle dealt round-robin to the 16 warps;
//   (4) back substitution per block in registers: shuffle + FMA per unknown.
// A is (d+1) x (d+1) with row pitch d+1 (fp64, shared memory); row d = r^T.  U: (d+1) x 16 panel scratch.
constexpr int kNB = 16;
constexpr int kCholThreads = 512;
constexpr int kUPitch = kNB + 1;

// Refinement mode (REFINE, b2_fit_refined): the right-hand side is g - alpha beta from rf (ctx->refine) instead of r from S,
// so the same factor of A + alpha I gives the correction dbeta; refine_update then moves the state.
__device__ void refine_update(const double* S, int d, int fit_intercept, bool singular, const double* dbeta, double* misc,
                              double* __restrict__ rf, double* __restrict__ out);

template <bool REFINE>
__global__ void __launch_bounds__(kCholThreads, 1)
solve_cholesky_kernel(double* S, int d, double alpha, int fit_intercept, double* __restrict__ out, const SolveXchg xc,
                      double* __restrict__ rf) {
  extern __shared__ double sm[];
  const int pitch = d + 1;
  double* A = sm;                        // rows 0..d-1 = A, row d = r^T
  double* r = A + d * pitch;             // alias of row d
  double* mean = A + (d + 1) * pitch;    // d
  double* invd = mean + d;               // d: 1 / D[k]
  double* misc = invd + d;               // [0] ybar, [1] max diag, [2] info (1-based failing pivot, 0 = ok)
  double* U = misc + 8;                  // (d+1) x kUPitch: unscaled panel entries of the current block column
  const int tid = threadIdx.x, lane = tid & 31;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);   // provably warp-uniform
  long long tm[5] = {0, 0, 0, 0, 0};     // phase cycle counters: build, diag, panel, update, backward
  long long tc0 = clock64();
  if (xc.own != nullptr) {
    // fused fit: this rank's partial S went to every peer from the Gram kernel's fold; gather = wait + sum, here
    __shared__ int ok;
    if (tid == 0) ok = xchg_wait(xc.own, xc.n_ranks, xc.epoch, xc.timeout_ns) ? 1 : 0;
    __syncthreads();
    if (!ok) {
      if (tid == 0) {
        xchg_flags(xc.own)[kXchgStatusWord] = xc.epoch;
        out[kOutInfo] = -1.0;             // the host turns this into B2_E_COMM (never a fit on a partial statistic)
      }
      return;
    }
    const int dp = d + 2;
    for (int base = 0; base < dp * dp; base += 4 * blockDim.x) {      // 4 elements x n_ranks loads in flight per thread
      double sv[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int idx = base + u * blockDim.x + tid;
        sv[u] = idx < dp * dp ? xchg_sum(xc.own, xc.n_ranks, xc.epoch, idx) : 0.0;
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int idx = base + u * blockDim.x + tid;
        if (idx < dp * dp) S[idx] = sv[u];
      }
    }
    __threadfence();
    __syncthreads();
  }
  build_normal_equations(S, d, alpha, fit_intercept, A, r, mean, &misc[0]);
  if constexpr (REFINE) {
    if (tid < d) r[tid] = rf[kRfGrad + tid] - alpha * rf[kRfBeta + tid];
    __syncthreads();
  }
  tm[0] = clock64() - tc0;
  if (warp == 0) {
    double mx = 0.0;
    for (int i = lane; i < d; i += 32) mx = fmax(mx, A[i * pitch + i]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (lane == 0) { misc[1] = mx; misc[2] = 0.0; }
  }
  __syncthreads();
  const double tiny = misc[1] * 1e-12;
  const int rows = d + 1;                // including the augmented row

  for (int kb = 0; kb < d; kb += kNB) {
    const int nb = (d - kb) < kNB ? (d - kb) : kNB;
    tc0 = clock64();
    // ---- (1) diagonal block: one warp, lane = (row, column parity): 16 rows x 2 halves, 8 columns per lane ----------
    if (warp == 0) {
      const int lrow = lane & (kNB - 1), h = lane >> 4;
      const bool act = lrow < nb;
      const int row = kb + (act ? lrow : 0);
      double a[kNB / 2];                                  // a[cc] = A[row][kb + 2 cc + h]; only columns <= row are meaningful
#pragma unroll
      for (int cc = 0; cc < kNB / 2; ++cc) {
        const int c = 2 * cc + h;
        a[cc] = (act && c < nb) ? A[row * pitch + kb + c] : 0.0;
      }
      double my_rc = 1.0;
      int first_bad = 0;
#pragma unroll
      for (int k = 0; k < kNB; ++k) {
        if (k < nb) {                                     // warp-uniform
          const int hk = k & 1, kk = k >> 1;              // column k lives in a[kk] of the lanes of half hk
          const double colk = a[kk];
          const double piv = __shfl_sync(0xffffffffu, colk, k | (hk << 4));
          const bool bad = !(piv > tiny);
          const double rc = bad ? 1.0 : rcp_pos(piv);
          const double u = __shfl_sync(0xffffffffu, colk, lrow | (hk << 4));   // u_ik = m_ik D_k of this lane's row
          my_rc = (lrow == k) ? rc : my_rc;
          first_bad = (bad && first_bad == 0) ? (kb + k + 1) : first_bad;
#pragma unroll
          for (int cc = 0; cc < kNB / 2; ++cc) {
            if (2 * cc + 1 > k) {                         // compile time: some column of this slot is right of the pivot
              const int c = 2 * cc + h;
              const double uc = __shfl_sync(0xffffffffu, colk, c | (hk << 4));   // u_ck
              if (c > k) a[cc] = fma(-(u * uc), rc, a[cc]);                      // a_ic -= u_ik u_ck / D_k
            }
          }
          if (h == hk && act && lrow > k) {               // column k of the rows below the pivot: multiplier and raw entry
            A[row * pitch + kb + k] = u * rc;
            U[row * kUPitch + k] = u;
          }
        }
      }
      if (act && h == 0) invd[kb + lrow] = my_rc;
      if (lane == 0 && first_bad != 0 && misc[2] == 0.0) misc[2] = (double)first_bad;
    }
    __syncthreads();
    tm[1] += clock64() - tc0; tc0 = clock64();
    if (misc[2] != 0.0) break;
    // ---- (2) panel: rows below the block (incl. the r row), 4 lanes per row (lane q owns columns c = q mod 4) ---------
    {
      const int prow = tid >> 2, q = tid & 3;
      const int below = rows - kb - nb;                   // <= 113 <= blockDim / 4
      const bool live = prow < below;
      const int i = kb + nb + (live ? prow : 0);
      double sv[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int c = 4 * j + q;
        sv[j] = (live && c < nb) ? A[i * pitch + kb + c] : 0.0;
      }
      const int qbase = lane & ~3;
      double rinv[kNB];                                   // 1 / D of the block: loaded once, off the chain
#pragma unroll
      for (int m = 0; m < kNB; ++m) rinv[m] = m < nb ? invd[kb + m] : 0.0;
      double out_m[4], out_u[4];                          // this lane's results (columns m = 4 j + q), stored after the
#pragma unroll                                            // loop so that the loads of U below are free to move up
      for (int j = 0; j < 4; ++j) { out_m[j] = 0.0; out_u[j] = 0.0; }
#pragma unroll
      for (int m = 0; m < kNB; ++m) {
        if (m < nb) {                                     // block-uniform
          const double um = __shfl_sync(0xffffffffu, sv[m >> 2], qbase | (m & 3));
          const double xm = um * rinv[m];
          if (q == (m & 3)) { out_m[m >> 2] = xm; out_u[m >> 2] = um; }
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            if (4 * j + 3 > m) {                          // compile time
              const int c = 4 * j + q;
              if (c > m && c < nb) sv[j] = fma(-xm, U[(kb + c) * kUPitch + m], sv[j]);
            }
          }
        }
      }
      if (live) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int m = 4 * j + q;
          if (m < nb) { A[i * pitch + kb + m] = out_m[j]; U[i * kUPitch + m] = out_u[j]; }
        }
      }
    }
    __syncthreads();
    tm[2] += clock64() - tc0; tc0 = clock64();
    // ---- (3) trailing update A[i][j] -= sum_m M[i][m] U[j][m] on the fp64 tensor-core path -----------------------------
    // 8 x 8 tiles of the lower triangle (i up to the r row), one DMMA m8n8k4 per 4 columns of the panel; a warp takes
    // every 16th tile.  Fragments (PTX mma.m8n8k4.f64): A row = lane / 4, col = lane % 4; B row(k) = lane % 4,
    // col(n) = lane / 4; C row = lane / 4, cols = 2 (lane % 4) + {0, 1}.
    {
      const int base = kb + nb;
      const int nti = (rows - base + 7) >> 3, ntj = (d - base + 7) >> 3;
      const int tri = ntj * (ntj + 1) / 2;
      const int total = tri + (nti > ntj ? ntj : 0);      // the r row may start one more tile row
      const int g = lane >> 2, t4 = lane & 3;
      constexpr int kWarps = kCholThreads / 32, kInFlight = 4;
      for (int t0 = warp; t0 < total; t0 += kWarps * kInFlight) {     // kInFlight independent tiles per pass: the loads and
        int ia[kInFlight], jb[kInFlight];                             // the 4-deep DMMA chains of the tiles overlap
        double c0[kInFlight], c1[kInFlight], av[kInFlight][kNB / 4], bv[kInFlight][kNB / 4];
#pragma unroll
        for (int f = 0; f < kInFlight; ++f) {
          const int t = t0 + f * kWarps;
          int ti = 0, tj = 0;
          if (t < tri) {
            ti = (int)((sqrtf(8.0f * (float)t + 1.0f) - 1.0f) * 0.5f);
            while (ti * (ti + 1) / 2 > t) --ti;
            while ((ti + 1) * (ti + 2) / 2 <= t) ++ti;
            tj = t - ti * (ti + 1) / 2;
          } else if (t < total) {
            ti = ntj; tj = t - tri;
          }
          const bool live = t < total;
          ia[f] = live ? base + 8 * ti + g : rows;                    // out of range: loads give 0, nothing is stored
          jb[f] = live ? base + 8 * tj + g : d;
#pragma unroll
          for (int sgm = 0; sgm < kNB / 4; ++sgm) {
            const int m = 4 * sgm + t4;
            av[f][sgm] = (ia[f] < rows && m < nb) ? -A[ia[f] * pitch + kb + m] : 0.0;
            bv[f][sgm] = (jb[f] < d && m < nb) ? U[jb[f] * kUPitch + m] : 0.0;
          }
          c0[f] = 0.0; c1[f] = 0.0;
        }
#pragma unroll
        for (int sgm = 0; sgm < kNB / 4; ++sgm) {
#pragma unroll
          for (int f = 0; f < kInFlight; ++f)
            asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
                         : "+d"(c0[f]), "+d"(c1[f]) : "d"(av[f][sgm]), "d"(bv[f][sgm]));
        }
#pragma unroll
        for (int f = 0; f < kInFlight; ++f) {
          const int jc = jb[f] - g + 2 * t4;
          if (ia[f] < rows) {
            if (jc < d) A[ia[f] * pitch + jc] += c0[f];
            if (jc + 1 < d) A[ia[f] * pitch + jc + 1] += c1[f];
          }
        }
      }
    }
    __syncthreads();
    tm[3] += clock64() - tc0;
  }
  tc0 = clock64();
  const bool singular = misc[2] != 0.0;
  if (!singular) {
    // row d now holds w = D^-1 M^-1 r.  backward: M^T b = w (unit diagonal), blocked from the bottom
    for (int kb = ((d - 1) / kNB) * kNB; kb >= 0; kb -= kNB) {
      const int nb = (d - kb) < kNB ? (d - kb) : kNB;
      if (warp == 0) {
        const int col = lane & (kNB - 1);
        const bool act = lane < nb;
        double lt[kNB];                                // lt[k] = M[kb+k][kb+col], k > col
#pragma unroll
        for (int k = 0; k < kNB; ++k) lt[k] = (act && k < nb && k > col) ? A[(kb + k) * pitch + kb + col] : 0.0;
        double z = act ? r[kb + col] : 0.0;
#pragma unroll
        for (int k = kNB - 1; k >= 0; --k) {
          if (k < nb) {
            const double bk = __shfl_sync(0xffffffffu, z, k);   // lane k is final: every i > k has been subtracted
            z = (lane < k) ? fma(-lt[k], bk, z) : z;
          }
        }
        __syncwarp();
        if (act) r[kb + lane] = z;
      }
      __syncthreads();
      for (int i = tid; i < kb; i += blockDim.x) {
        double acc0 = 0.0, acc1 = 0.0;
#pragma unroll
        for (int m = 0; m < kNB; m += 2) {
          if (m < nb) acc0 = fma(A[(kb + m) * pitch + i], r[kb + m], acc0);
          if (m + 1 < nb) acc1 = fma(A[(kb + m + 1) * pitch + i], r[kb + m + 1], acc1);
        }
        r[i] -= acc0 + acc1;
      }
      __syncthreads();
    }
  }
  tm[4] = clock64() - tc0;
  if constexpr (REFINE) {
    refine_update(S, d, fit_intercept, singular, r, misc, rf, out);
    return;
  }
  if (tid == 0)
    for (int k = 0; k < 5; ++k) out[kOutSingular + k] = (double)tm[k];
  for (int i = tid; i < d; i += blockDim.x) out[i] = singular ? 0.0 : r[i];
  if (warp == 0) {
    double part = 0.0;
    for (int i = lane; i < d; i += 32) part += mean[i] * r[i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
    if (lane == 0) {
      out[kOutIntercept] = singular ? 0.0 : misc[0] - part;
      out[kOutInfo] = misc[2];
    }
  }
}

// step = max_j |dbeta_j| sigma_j / sigma_y, sigma from S's centred diagonal.  A step above the last kept one means the last
// kept correction left a larger error than it found (the next correction estimates what the previous one left), so the
// state returns to before it and the pass reports the guard (out[kOutRefineGuard] = 1); so does a non-finite correction
// or a failed factorisation.  Otherwise beta += dbeta, b0' += g_1 / n.  out: coef = beta, intercept = b0' - m.beta.
__device__ void refine_update(const double* S, int d, int fit_intercept, bool singular, const double* dbeta, double* misc,
                              double* __restrict__ rf, double* __restrict__ out) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int dp = d + 2;
  const double n = __ldcg(S + d * dp + d);
  if (warp == 0) {
    double mx = 0.0;
    bool finite = true;
    for (int i = lane; i < d; i += 32) {
      const double sx = __ldcg(S + i * dp + d);
      const double c = __ldcg(S + i * dp + i) - sx * (sx / n);
      mx = fmax(mx, fabs(dbeta[i]) * sqrt(fmax(c, 0.0)));
      finite = finite && isfinite(dbeta[i]);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    finite = __all_sync(0xffffffffu, finite) && isfinite(rf[kRfGrad + kMaxD]);
    if (lane == 0) {
      const double sy = __ldcg(S + d * dp + d + 1);
      const double cy = __ldcg(S + (d + 1) * dp + d + 1) - sy * (sy / n);
      const double sig = sqrt(fmax(cy, 0.0));
      const double step = sig > 0.0 ? mx / sig : mx;
      misc[3] = step;
      misc[4] = (singular || !finite || !(step <= rf[kRfStep])) ? 1.0 : 0.0;
    }
  }
  __syncthreads();
  const bool guard = misc[4] != 0.0;
  for (int i = tid; i < d; i += blockDim.x) {
    const double b = rf[kRfBeta + i];
    if (guard) {
      rf[kRfBeta + i] = rf[kRfPrevBeta + i];
    } else {
      rf[kRfPrevBeta + i] = b;
      rf[kRfBeta + i] = b + dbeta[i];
    }
  }
  if (tid == 0) {
    const double b0 = rf[kRfB0];
    if (guard) {
      rf[kRfB0] = rf[kRfPrevB0];
    } else {
      rf[kRfPrevB0] = b0;
      rf[kRfB0] = fit_intercept ? b0 + rf[kRfGrad + kMaxD] / n : b0;
      rf[kRfStep] = misc[3];
    }
  }
  __syncthreads();
  for (int i = tid; i < d; i += blockDim.x) out[i] = rf[kRfBeta + i];
  if (warp == 0) {
    double part = 0.0;
    for (int i = lane; i < d; i += 32) part += rf[kRfMean + i] * rf[kRfBeta + i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
    if (lane == 0) {
      out[kOutIntercept] = rf[kRfB0] - part;
      out[kOutInfo] = misc[2];
      out[kOutRefineStep] = misc[3];
      out[kOutRefineGuard] = misc[4];
    }
  }
}

// pair (p, q) of slot k in round `round` of the round-robin tournament over m (even) players
__device__ __forceinline__ void rr_pair(int m, int round, int k, int* p, int* q) {
  const int mm = m - 1;
  int a, b;
  if (k == 0) { a = mm; b = round % mm; }
  else { a = (round + k) % mm; b = (round - k + mm) % mm; }
  *p = a < b ? a : b;
  *q = a < b ? b : a;
}

__global__ void __launch_bounds__(512, 1)
solve_spectral_kernel(const double* __restrict__ S, int d, double cond, int fit_intercept,
                      double* __restrict__ out) {
  extern __shared__ double sm[];
  const int pitch = d + 1;
  double* W = sm;                  // W^T: W[col * pitch + row]   (A is symmetric, so W0 = A either way)
  double* r = W + d * pitch;
  double* mean = r + d;
  double* lam = mean + d;          // column norms
  double* misc = lam + d;          // [0] ybar
  __shared__ int rotated;
  build_normal_equations(S, d, 0.0, fit_intercept, W, r, mean, &misc[0]);

  const int m = d + (d & 1);       // even player count; player d (if any) is a phantom
  const int pairs = m / 2;
  const int sub = threadIdx.x & 7; // 8 threads cooperate on one pair
  const int slot0 = threadIdx.x >> 3;
  for (int sweep = 0; sweep < 24 && d > 1; ++sweep) {
    if (threadIdx.x == 0) rotated = 0;
    __syncthreads();
    for (int round = 0; round < m - 1; ++round) {
      for (int slot = slot0; slot < ((pairs + 63) / 64) * 64; slot += 64) {
        int p = 0, q = 0;
        const bool live_slot = slot < pairs;
        if (live_slot) rr_pair(m, round, slot, &p, &q);
        const bool live = live_slot && q < d;
        double a = 0.0, b = 0.0, g = 0.0;
        if (live) {
          for (int row = sub; row < d; row += 8) {
            const double wp = W[p * pitch + row], wq = W[q * pitch + row];
            a += wp * wp; b += wq * wq; g += wp * wq;
          }
        }
#pragma unroll
        for (int o = 1; o < 8; o <<= 1) {
          a += __shfl_xor_sync(0xffffffffu, a, o);
          b += __shfl_xor_sync(0xffffffffu, b, o);
          g += __shfl_xor_sync(0xffffffffu, g, o);
        }
        if (live && fabs(g) > 1e-15 * sqrt(a * b) && a * b > 0.0) {
          const double zeta = (b - a) / (2.0 * g);
          const double t = (zeta >= 0.0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
          const double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
          for (int row = sub; row < d; row += 8) {
            const double wp = W[p * pitch + row], wq = W[q * pitch + row];
            W[p * pitch + row] = c * wp - s * wq;
            W[q * pitch + row] = s * wp + c * wq;
          }
          if (sub == 0 && fabs(g) > 1e-13 * sqrt(a * b)) rotated = 1;
        }
      }
      __syncthreads();
    }
    if (!rotated) break;
    __syncthreads();
  }
  // |eigenvalues| = column norms.  The sign is lost in W^T W = V A^2 V^T; it comes back from lambda_k^3 = w_k^T A w_k,
  // with A formed again from S exactly as build_normal_equations formed it (one warp per column, lane = row of A w_k).
  // A centred Gram that rounding has made slightly indefinite then reports its negative eigenvalues as 0, as the
  // eigenvalue kernel and sklearn's gelsd (singular values of the centred rows) do: they are not counted in rank_ and
  // give no term of the minimum-norm solution.
  {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5, dp = d + 2;
    const double n = __ldcg(S + d * dp + d);
    for (int k = warp; k < d; k += nwarps) {
      const double* w = W + k * pitch;
      double s2 = 0.0, cube = 0.0;
      for (int i = lane; i < d; i += 32) {
        double aw = 0.0;
        for (int j = 0; j < d; ++j) aw = fma(__ldcg(S + i * dp + j) - n * mean[i] * mean[j], w[j], aw);
        s2 = fma(w[i], w[i], s2);
        cube = fma(w[i], aw, cube);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        s2 += __shfl_xor_sync(0xffffffffu, s2, o);
        cube += __shfl_xor_sync(0xffffffffu, cube, o);
      }
      if (lane == 0) lam[k] = cube > 0.0 ? sqrt(s2) : 0.0;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    // descending singular values (selection sort on a copy in `out`), rank, min-norm coefficients
    double mx = 0.0;
    for (int k = 0; k < d; ++k) mx = fmax(mx, lam[k]);
    const double smax = sqrt(mx);
    int rank = 0;
    for (int k = 0; k < d; ++k) {
      out[kOutSingular + k] = sqrt(lam[k]);
      if (sqrt(lam[k]) > cond * smax) ++rank;
    }
    for (int i = 0; i < d; ++i) {
      int best = i;
      for (int j = i + 1; j < d; ++j) if (out[kOutSingular + j] > out[kOutSingular + best]) best = j;
      const double tmp = out[kOutSingular + i];
      out[kOutSingular + i] = out[kOutSingular + best];
      out[kOutSingular + best] = tmp;
    }
    out[kOutRank] = (double)rank;
    misc[1] = smax;
  }
  __syncthreads();
  const double smax = misc[1];
  // coef = sum_k w_k (w_k . r) / lambda_k^3 over kept k
  for (int k = threadIdx.x; k < d; k += blockDim.x) {
    double dot = 0.0;
    for (int row = 0; row < d; ++row) dot += W[k * pitch + row] * r[row];
    const bool keep = sqrt(lam[k]) > cond * smax && lam[k] > 0.0;
    lam[k] = keep ? dot / (lam[k] * lam[k] * lam[k]) : 0.0;  // reuse lam as the per-column weight
  }
  __syncthreads();
  for (int i = threadIdx.x; i < d; i += blockDim.x) {
    double b = 0.0;
    for (int k = 0; k < d; ++k) b += W[k * pitch + i] * lam[k];
    r[i] = b;
    out[i] = b;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double b0 = misc[0];
    for (int i = 0; i < d; ++i) b0 -= mean[i] * r[i];
    out[kOutIntercept] = b0;
    out[kOutInfo] = 0.0;
  }
}

// ---- eigenvalues only: singular_ and rank_ of the fitted estimator -------------------------------------------------
// LinearRegression.fit stores `singular_` (singular values of the centred X, descending) and `rank_` next to the
// coefficients (sklearn/linear_model/_base.py: `self.coef_, _, self.rank_, self.singular_ = linalg.lstsq(...)`), and the
// joblib artefact of stage_1_train_model.py:113-114 carries them.  They are sqrt(eig(Xc^T Xc)), i.e. eigenvalues of the
// same centred Gram matrix the Cholesky solve factors -- no eigenvectors are needed unless the matrix is rank deficient
// (then solve_spectral_kernel computes the minimum-norm coefficients).  One CTA:
//   (a) Householder tridiagonalisation T = Q^T A Q in shared memory (d - 2 reflections; matvec + rank-2 update by all
//       threads, 3 block syncs per reflection);
//   (b) eigenvalues of T by multisection on Sturm counts: 4 threads per eigenvalue evaluate the division-free
//       characteristic-polynomial recurrence (one dependent FMA per row, power-of-two rescaling every 8 rows) at the 4
//       interior points of its bracket, so every round shrinks every bracket 5x with no block-level synchronisation.
constexpr int kEigThreads = 512;
constexpr int kEigCols = kMaxD / 4;      // columns per thread: thread (row, q) keeps A[row][4 jj + q] in registers
constexpr int kEigRounds = 24;           // 5-section rounds: 5^24 = 6e16 > 2^53 * the 1.002 initial bracket

// number of eigenvalues of T below x = sign changes of p_0 = 1, p_1 = d_0 - x, p_i = (d_{i-1} - x) p_{i-1} - e_{i-2}^2 p_{i-2}.
// dp8 = d rounded up to 8; rows d .. dp8-1 are decoupled 1 x 1 blocks far above the spectrum (no sign change).  Unrolled
// by 8: the loads of a group do not depend on the recurrence, the chain is one FMA (+ the zero test) per row.
__device__ __forceinline__ int sturm_count(const double* __restrict__ dd, const double* __restrict__ ee2, int dp8, double x) {
  double pm = 1.0, p = dd[0] - x;
  if (p == 0.0) p = -1e-300;
  int count = p < 0.0 ? 1 : 0;
  double eprev = 0.0;                                                                   // e_{i-1}^2 of the row before the group
  for (int i0 = 0; i0 < dp8; i0 += 8) {
    double dv[8], ev[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) { dv[u] = dd[i0 + u] - x; ev[u] = ee2[i0 + u]; }     // ee2[i] couples rows i and i + 1
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      if (i0 + u > 0) {                                                                 // row 0 is p_1 above
        double pn = fma(dv[u], p, -((u == 0 ? eprev : ev[u - 1]) * pm));
        // sign change / exact zero on the integer pipe (the fp64 pipe is the bottleneck of this loop): a zero counts
        // as a sign change and continues as a tiny value of the opposite sign
        const int hn = __double2hiint(pn), hp = __double2hiint(p);
        if (((hn & 0x7fffffff) | __double2loint(pn)) == 0) pn = __hiloint2double((~hp & 0x80000000) | 0x01a00000, 0);
        count += (int)(((unsigned int)(__double2hiint(pn) ^ hp)) >> 31);
        pm = p; p = pn;
      }
    }
    eprev = ev[7];
    const int eb = (__double2hiint(p) >> 20) & 0x7ff;                                   // keep the pair in range: 2^-exponent(p)
    int sh = 1023 - eb;
    sh = sh > 1000 ? 1000 : (sh < -1000 ? -1000 : sh);
    const double sc = __hiloint2double((1023 + sh) << 20, 0);
    p *= sc; pm *= sc;
  }
  return count;
}

__global__ void __launch_bounds__(kEigThreads, 1)
solve_eigvals_kernel(const double* S, int d, double cond, int fit_intercept, double* __restrict__ out) {
  extern __shared__ __align__(16) double sm[];
  const int pitch = d + 1;
  double* A = sm;                         // symmetric, full storage; lives in registers during the tridiagonalisation
  double* r = A + d * pitch;              // (unused here; build_normal_equations fills it)
  double* mean = A + (d + 1) * pitch;
  double* misc = mean + 2 * d;
  // [2][kMaxD]: (v_j, w_j) of the current reflection, by step parity; 16-byte aligned (the offset in doubles made even)
  double2* vw = reinterpret_cast<double2*>(sm + ((((size_t)(misc + 8 - sm)) + 1) & ~(size_t)1));
  double* pv = reinterpret_cast<double*>(vw + 2 * kMaxD);   // [kMaxD] tau * A v
  double* dd = pv + kMaxD;                // [kMaxD + 8] diagonal of T (padded for the unrolled Sturm recurrence)
  double* ee2 = dd + kMaxD + 8;           // [kMaxD + 8] squared off-diagonal of T
  double* lam = ee2 + kMaxD + 8;          // [kMaxD] eigenvalues, ascending
  const int tid = threadIdx.x, lane = tid & 31;
  long long tph[4];
  long long tq = clock64();
  build_normal_equations(S, d, 0.0, fit_intercept, A, r, mean, &misc[0]);
  tph[0] = clock64() - tq; tq = clock64();

  // ---- (a) Householder tridiagonalisation, the matrix in registers: thread (row, q) owns columns j = 4 jj + q ----------
  const int row = tid >> 2, q = tid & 3;
  double a[kEigCols];
#pragma unroll
  for (int jj = 0; jj < kEigCols; ++jj) {
    const int j = 4 * jj + q;
    a[jj] = (row < d && j < d) ? A[row * pitch + j] : 0.0;
  }
  for (int j = tid; j < 2 * kMaxD; j += blockDim.x) vw[j] = make_double2(0.0, 0.0);
  for (int j = tid; j < kMaxD; j += blockDim.x) pv[j] = 0.0;
  __syncthreads();
  for (int k = 0; k + 2 < d; ++k) {
    double2* vwk = vw + (k & 1) * kMaxD;
    // (a1) the reflector of column k, by the 4 threads that own row k (= column k, the matrix is symmetric):
    //      x = A[k][k+1 ..]; beta = -sign(x0) |x|, tau = (beta - x0) / beta, v = x / (x0 - beta), v[k+1] = 1
    if (row == k) {
      const unsigned int qmask = 0xFu << (lane & ~3);
      double s2p[4] = {0.0, 0.0, 0.0, 0.0};
#pragma unroll
      for (int jj = 0; jj < kEigCols; ++jj) {
        const int j = 4 * jj + q;
        if (j > k + 1) s2p[jj & 3] = fma(a[jj], a[jj], s2p[jj & 3]);
        if (j == k + 1) misc[6] = a[jj];
        if (j == k) misc[7] = a[jj];
      }
      double s2 = (s2p[0] + s2p[1]) + (s2p[2] + s2p[3]);
      s2 += __shfl_xor_sync(qmask, s2, 1);
      s2 += __shfl_xor_sync(qmask, s2, 2);
      __syncwarp(qmask);
      const double x0 = misc[6];
      double tau = 0.0, beta = x0, scale = 0.0;
      if (s2 > 0.0) {
        const double nrm = sqrt(fma(x0, x0, s2));
        beta = x0 >= 0.0 ? -nrm : nrm;
        tau = (beta - x0) / beta;
        scale = 1.0 / (x0 - beta);
      }
#pragma unroll
      for (int jj = 0; jj < kEigCols; ++jj) {
        const int j = 4 * jj + q;
        if (j < d) vwk[j].x = (j > k + 1) ? a[jj] * scale : (j == k + 1 ? 1.0 : 0.0);
      }
      if (q == 0) { misc[1] = tau; dd[k] = misc[7]; ee2[k] = beta * beta; }
    }
    __syncthreads();
    const double tau = misc[1];
    if (tau != 0.0) {                     // block-uniform
      // The fp64 pipe is what this phase runs on, so finished rows and columns are
      // skipped, not multiplied by zero: a warp whose 8 rows are all <= k does nothing, a 32-column group <= k is
      // jumped over (warp-uniform tests; the register-resident matrix needs compile-time column indices).
      const bool warp_live = ((tid >> 5) * 8 + 7) > k;
      // (a2) p = tau * A v
      if (warp_live) {
        double acc0 = 0.0, acc1 = 0.0, acc2 = 0.0, acc3 = 0.0;
#pragma unroll
        for (int b = 0; b < kEigCols / 8; ++b) {
          if (32 * b + 31 > k) {
#pragma unroll
            for (int u = 0; u < 8; u += 4) {
              const int jj = 8 * b + u;
              acc0 = fma(a[jj], vwk[4 * jj + q].x, acc0);
              acc1 = fma(a[jj + 1], vwk[4 * (jj + 1) + q].x, acc1);
              acc2 = fma(a[jj + 2], vwk[4 * (jj + 2) + q].x, acc2);
              acc3 = fma(a[jj + 3], vwk[4 * (jj + 3) + q].x, acc3);
            }
          }
        }
        double acc = (acc0 + acc1) + (acc2 + acc3);
        acc += __shfl_xor_sync(0xffffffffu, acc, 1);
        acc += __shfl_xor_sync(0xffffffffu, acc, 2);
        if (q == 0) pv[row] = (row > k && row < d) ? tau * acc : 0.0;
      } else if (q == 0) {
        pv[row] = 0.0;
      }
      __syncthreads();
      // (a3) K = -tau/2 (p . v), recomputed by every warp; w = p + K v is formed on the fly in (a4) -- one more FMA per
      // element, one block barrier and one shared-memory round trip fewer per reflection (the loop is latency bound)
      double dot = 0.0;
#pragma unroll
      for (int u = 0; u < kMaxD / 32; ++u) dot = fma(pv[lane + 32 * u], vwk[lane + 32 * u].x, dot);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
      const double K = -0.5 * tau * dot;
      // (a4) A -= v w^T + w v^T: rows and columns up to k have v = w = 0 and keep their values
      if (warp_live) {
        const double vr = vwk[row].x, wr = fma(K, vr, pv[row]);
#pragma unroll
        for (int b = 0; b < kEigCols / 8; ++b) {
          if (32 * b + 31 > k) {
#pragma unroll
            for (int u = 0; u < 8; ++u) {
              const int jj = 8 * b + u;
              const double vj = vwk[4 * jj + q].x, wj = fma(K, vj, pv[4 * jj + q]);
              a[jj] = fma(-vr, wj, fma(-wr, vj, a[jj]));
            }
          }
        }
      }
    }
  }
  // the last 2 x 2 block comes from the registers of rows d-2, d-1
  __syncthreads();
  tph[1] = clock64() - tq; tq = clock64();
  if (row < d && row + 2 >= d) {
#pragma unroll
    for (int jj = 0; jj < kEigCols; ++jj) {
      const int j = 4 * jj + q;
      if (j < d && j + 2 >= d) A[row * pitch + j] = a[jj];
    }
  }
  __syncthreads();
  const int dp8 = (d + 7) & ~7;
  if (tid == 0) {
    if (d >= 2) { dd[d - 2] = A[(d - 2) * pitch + d - 2]; ee2[d - 2] = A[(d - 1) * pitch + d - 2] * A[(d - 1) * pitch + d - 2]; }
    dd[d - 1] = A[(d - 1) * pitch + d - 1];
  }
  __syncthreads();
  // Gershgorin interval (one row per thread, warp 0..3 then a 4-entry combine), then a power-of-two scaling so that
  // |d_i - x| <= 2 and e_i^2 <= 1 in the recurrence
  {
    double glo = 1e300, ghi = -1e300;
    if (tid < d) {
      const double rad = (tid > 0 ? sqrt(ee2[tid - 1]) : 0.0) + (tid + 1 < d ? sqrt(ee2[tid]) : 0.0);
      glo = dd[tid] - rad; ghi = dd[tid] + rad;
    }
    if (tid < kMaxD) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        glo = fmin(glo, __shfl_xor_sync(0xffffffffu, glo, o));
        ghi = fmax(ghi, __shfl_xor_sync(0xffffffffu, ghi, o));
      }
      if (lane == 0) { pv[2 * (tid >> 5)] = glo; pv[2 * (tid >> 5) + 1] = ghi; }
    }
  }
  __syncthreads();
  if (tid == 0) {
    double glo = pv[0], ghi = pv[1];
    for (int w = 1; w < kMaxD / 32; ++w) { glo = fmin(glo, pv[2 * w]); ghi = fmax(ghi, pv[2 * w + 1]); }
    const double span = fmax(fmax(fabs(glo), fabs(ghi)), 1e-300);
    int ex = ((__double2hiint(span) >> 20) & 0x7ff) - 1023 + 1;
    ex = ex > 1000 ? 1000 : (ex < -1000 ? -1000 : ex);
    misc[2] = __hiloint2double((1023 - ex) << 20, 0);   // 2^-ex
    misc[3] = __hiloint2double((1023 + ex) << 20, 0);   // 2^ex
    misc[4] = glo; misc[5] = ghi;
  }
  __syncthreads();
  const double sdown = misc[2], sup = misc[3];
  for (int i = tid; i < dp8; i += blockDim.x) {
    if (i < d) { dd[i] *= sdown; ee2[i] = (i + 1 < d) ? ee2[i] * sdown * sdown : 0.0; }
    else { dd[i] = 8.0; ee2[i] = 0.0; }                 // padding rows: decoupled, above every scaled eigenvalue (|x| <= 1)
  }
  __syncthreads();
  tph[2] = clock64() - tq; tq = clock64();
  // (b) multisection: quad (4 consecutive lanes) owns eigenvalue index e; bracket invariant count(lo) <= e < count(hi)
  for (int e0 = 0; e0 < d; e0 += kEigThreads / 4) {
    const int e = e0 + (tid >> 2);
    const bool live = e < d;
    double lo = misc[4] * sdown, hi = misc[5] * sdown;
    const double w0 = hi - lo;
    lo -= 1e-3 * w0 + 1e-300; hi += 1e-3 * w0 + 1e-300;
    for (int round = 0; round < kEigRounds; ++round) {
      const double step = (hi - lo) * 0.2;
      const double x = lo + step * (double)(q + 1);
      const int c = live ? sturm_count(dd, ee2, dp8, x) : 0;
      const bool below = c <= e;                       // x is still a lower bound of eigenvalue e
      // the 4 points are increasing in q: new lo = the last `below` point, new hi = the first non-`below` point
      const unsigned int quad_shift = (unsigned int)(lane & ~3);
      const unsigned int bal = (__ballot_sync(0xffffffffu, below) >> quad_shift) & 0xFu;
      const int nbel = __popc(bal);                    // below is monotone in x: the first nbel points are lower bounds
      const double nlo = nbel > 0 ? lo + step * (double)nbel : lo;
      const double nhi = nbel < 4 ? lo + step * (double)(nbel + 1) : hi;
      lo = nlo; hi = nhi;
    }
    if (live && q == 0) lam[e] = 0.5 * (lo + hi) * sup;
  }
  __syncthreads();
  tph[3] = clock64() - tq;
  if (tid == 0)
    for (int k = 0; k < 4; ++k) out[kOutRows + 1 + k] = (double)tph[k];   // phase cycles (development builds print them)
  // singular values descending, rank = #{s > cond * s_max}
  const double lmax = fmax(lam[d - 1], 0.0);
  const double smax = sqrt(lmax);
  int rk = 0;
  for (int i = tid; i < d; i += blockDim.x) {
    const double sv = sqrt(fmax(lam[d - 1 - i], 0.0));
    out[kOutSingular + i] = sv;
    rk += (sv > cond * smax) ? 1 : 0;
  }
  __shared__ int rank_total;
  if (tid == 0) rank_total = 0;
  __syncthreads();
  if (rk) atomicAdd(&rank_total, rk);
  __syncthreads();
  if (tid == 0) {
    out[kOutRank] = (double)rank_total;
    out[kOutInfo] = 0.0;
    out[kOutRows] = S[d * (d + 2) + d];        // rows in the statistic: singular_ has min(rows, d) entries
  }
}

// ---- eigenvalues and orthonormal eigenvectors: b2_solve_eigh and the leave-one-out pass of b2_ridge_loo -------------
// The one-sided Jacobi above keeps only W = A V; normalising a column of W whose eigenvalue is near zero gives noise.
// Here two-sided cyclic Jacobi rotates A itself (packed upper triangle, 66 KB at D = 128) and accumulates V = the product
// of the rotations (131 KB), so V is orthonormal to working precision whatever the spectrum.  One round of the
// round-robin tournament (rr_pair) rotates m / 2 disjoint pairs at once: (1) each pair's (c, s) from its 2 x 2 diagonal
// block, (2) every 2 x 2 block of pairs (P1, P2) becomes J1^T B J2 in one step -- the blocks are disjoint, so no thread
// reads what another writes -- and the columns p, q of V rotate.  A pair rotates when |a_pq| > eps/2 sqrt(|a_pp a_qq|) and
// above 1e-20 of the largest diagonal entry; the sweeps stop after one without a rotation.  Cyclic Jacobi converges
// quadratically once the off-diagonal part is small; if kEighMaxSweeps sweeps still rotate, the kernel reports it (the
// host turns that into an error) instead of returning an unconverged Q.
// Output (ctx->loo): eigenvalues ascending, negative rounding values as 0; Q[i][k] (row pitch kMaxD), column k for
// eigenvalue k; the means m, ybar, n, h0 = 1 / n (0 without an intercept), c = Q^T r and whether the sweeps converged.
constexpr int kEighThreads = 512;
constexpr int kEighMaxSweeps = 30;

__host__ __device__ inline int eigh_m(int d) { return d + (d & 1); }
__device__ __forceinline__ int packed_ix(int i, int j) { return i <= j ? j * (j + 1) / 2 + i : i * (i + 1) / 2 + j; }

size_t eigh_smem_bytes(int d) {
  const size_t m = (size_t)eigh_m(d);
  const size_t full = (size_t)d * (d + 1) > m * m ? (size_t)d * (d + 1) : m * m;   // A (build) then V, same region
  return sizeof(double) * (m * (m + 1) / 2 + full + 3 * (size_t)kMaxD + 16 + 2 * (kMaxD / 2)) + sizeof(int) * kMaxD;
}

__global__ void __launch_bounds__(kEighThreads, 1)
solve_eigh_kernel(const double* __restrict__ S, int d, int fit_intercept, double* __restrict__ loo) {
  extern __shared__ double sm[];
  const int m = eigh_m(d), M = m / 2, pitch = d + 1;
  double* AP = sm;                                   // packed upper triangle of the m x m matrix (row/column d: phantom)
  double* V = AP + m * (m + 1) / 2;                  // V^T: V[k * m + i] = V_ik; first holds A (pitch d + 1) from the build
  const size_t full = (size_t)d * (d + 1) > (size_t)m * m ? (size_t)d * (d + 1) : (size_t)m * m;
  double* r = V + full;
  double* mean = r + kMaxD;
  double* lam = mean + kMaxD;
  double* misc = lam + kMaxD;                        // [0] ybar, [1] largest |diagonal|
  double* cs = misc + 16;                            // [kMaxD / 2] c, [kMaxD / 2] s of the current round
  int* pq = reinterpret_cast<int*>(cs + kMaxD);      // [kMaxD / 2] p | q << 16
  __shared__ int rotated, converged;
  const int tid = threadIdx.x;
  if (tid == 0) converged = d <= 1 ? 1 : 0;
  build_normal_equations(S, d, 0.0, fit_intercept, V, r, mean, &misc[0]);
  for (int t = tid; t < m * (m + 1) / 2; t += blockDim.x) AP[t] = 0.0;
  __syncthreads();
  for (int t = tid; t < d * d; t += blockDim.x) {
    const int i = t / d, j = t - i * d;
    if (i <= j) AP[packed_ix(i, j)] = V[i * pitch + j];
  }
  if (tid == 0) {
    double mx = 0.0;
    for (int i = 0; i < d; ++i) mx = fmax(mx, fabs(V[i * pitch + i]));
    misc[1] = mx;
  }
  __syncthreads();
  for (int t = tid; t < m * m; t += blockDim.x) V[t] = (t / m == t % m) ? 1.0 : 0.0;
  __syncthreads();
  const double floor_abs = 1e-20 * misc[1];
  constexpr double kHalfEps = 1.1102230246251565e-16;
  for (int sweep = 0; sweep < kEighMaxSweeps && d > 1; ++sweep) {
    if (tid == 0) rotated = 0;
    __syncthreads();
    for (int round = 0; round < m - 1; ++round) {
      // (1) the rotation of each pair
      if (tid < M) {
        int p, q;
        rr_pair(m, round, tid, &p, &q);
        const double app = AP[packed_ix(p, p)], aqq = AP[packed_ix(q, q)], apq = AP[packed_ix(p, q)];
        double c = 1.0, s = 0.0;
        if (fabs(apq) > floor_abs && fabs(apq) > kHalfEps * sqrt(fabs(app) * fabs(aqq))) {
          const double tau = (aqq - app) / (2.0 * apq);
          const double t = fabs(tau) > 1e150 ? 0.5 / tau
                                             : (tau >= 0.0 ? 1.0 : -1.0) / (fabs(tau) + sqrt(1.0 + tau * tau));
          c = 1.0 / sqrt(1.0 + t * t);
          s = t * c;
          rotated = 1;
        }
        cs[tid] = c;
        cs[kMaxD / 2 + tid] = s;
        pq[tid] = p | (q << 16);
      }
      __syncthreads();
      // (2) A <- J^T A J block by block, V <- V J
      for (int t = tid; t < M * M; t += blockDim.x) {
        const int P1 = t / M, P2 = t - P1 * M;
        if (P2 < P1) continue;
        const int p1 = pq[P1] & 0xffff, q1 = pq[P1] >> 16, p2 = pq[P2] & 0xffff, q2 = pq[P2] >> 16;
        const double c1 = cs[P1], s1 = cs[kMaxD / 2 + P1];
        if (P1 == P2) {
          if (s1 != 0.0) {
            const double app = AP[packed_ix(p1, p1)], aqq = AP[packed_ix(q1, q1)], apq = AP[packed_ix(p1, q1)];
            const double tt = s1 / c1;
            AP[packed_ix(p1, p1)] = app - tt * apq;
            AP[packed_ix(q1, q1)] = aqq + tt * apq;
            AP[packed_ix(p1, q1)] = 0.0;
          }
          continue;
        }
        const double c2 = cs[P2], s2 = cs[kMaxD / 2 + P2];
        if (s1 == 0.0 && s2 == 0.0) continue;
        const int i11 = packed_ix(p1, p2), i12 = packed_ix(p1, q2), i21 = packed_ix(q1, p2), i22 = packed_ix(q1, q2);
        const double x11 = AP[i11], x12 = AP[i12], x21 = AP[i21], x22 = AP[i22];
        const double u11 = c1 * x11 - s1 * x21, u12 = c1 * x12 - s1 * x22;     // rows: J1^T B
        const double u21 = s1 * x11 + c1 * x21, u22 = s1 * x12 + c1 * x22;
        AP[i11] = c2 * u11 - s2 * u12;                                          // columns: (J1^T B) J2
        AP[i12] = s2 * u11 + c2 * u12;
        AP[i21] = c2 * u21 - s2 * u22;
        AP[i22] = s2 * u21 + c2 * u22;
      }
      for (int t = tid; t < M * d; t += blockDim.x) {
        const int P = t / d, i = t - P * d;
        const double s = cs[kMaxD / 2 + P];
        if (s == 0.0) continue;
        const double c = cs[P];
        const int p = pq[P] & 0xffff, q = pq[P] >> 16;
        const double vp = V[p * m + i], vq = V[q * m + i];
        V[p * m + i] = c * vp - s * vq;
        V[q * m + i] = s * vp + c * vq;
      }
      __syncthreads();
    }
    if (!rotated) {
      if (tid == 0) converged = 1;
      break;
    }
    __syncthreads();
  }
  __syncthreads();
  // ascending order by rank (ties by index), negative rounding eigenvalues as 0; c = Q^T r
  for (int k = tid; k < d; k += blockDim.x) lam[k] = AP[packed_ix(k, k)];
  __syncthreads();
  const int dp = d + 2;
  const double n = __ldcg(S + d * dp + d);
  for (int k = tid; k < d; k += blockDim.x) {
    const double lk = lam[k];
    int rank = 0;
    for (int j = 0; j < d; ++j) rank += (lam[j] < lk || (lam[j] == lk && j < k)) ? 1 : 0;
    double ck = 0.0;
    for (int i = 0; i < d; ++i) {
      const double v = V[k * m + i];
      loo[kLooQ + i * kMaxD + rank] = v;
      ck = fma(v, r[i], ck);
    }
    loo[kLooLam + rank] = fmax(lk, 0.0);
    loo[kLooC + rank] = ck;
  }
  for (int i = tid; i < d; i += blockDim.x) loo[kLooMean + i] = mean[i];
  if (tid == 0) {
    loo[kLooMisc + 0] = misc[0];
    loo[kLooMisc + 1] = n;
    loo[kLooMisc + 2] = fit_intercept && n > 0.0 ? 1.0 / n : 0.0;
    loo[kLooMisc + 3] = converged ? 1.0 : 0.0;
  }
}

// ---- elastic net: a whole regularisation path by cyclic coordinate descent on the centred Gram (b2_solve_enet_path) --
//      and every (l1_ratio, fold) path of a cross-validation in one launch (b2_solve_enet_cv)
// Restates scikit-learn's enet_coordinate_descent_gram (sklearn/linear_model/_cd_fast.pyx) with enet_path's scaling
// (l1_reg = alpha l1_ratio n, l2_reg = alpha (1 - l1_ratio) n) and, without user alphas, its _alpha_grid.  Q, q come
// from build_normal_equations at alpha = 0; y_norm2 = S_yy - n ybar^2.  DESIGN.md section 7.
//   Constant columns: a column whose centred diagonal is not above kEnetConstCol times its raw one (standard deviation
//   <= 1e-6 of its root mean square, 16 fp32 ulps) has a centred Gram row and column of rounding noise; it is treated as
//   exactly constant -- Q row and column and q_j zeroed, coefficient 0, never updated -- which is what sklearn does for
//   Q_jj == 0 on exactly centred rows.
//   One warp runs everything after the build (the sweeps are one dependent chain): lane l holds (Qw, w, q, Q_jj and
//   1 / (Q_jj + l2_reg)) of features l + 32 u, so there is no division in the chain.  The step of coordinate j, formed by
//   its owner lane, goes to every lane by one shuffle and each lane applies its entries of Q's row j (shared memory).  The
//   active set is a 128-bit mask walked with __ffs inside a static loop over u, so the register arrays stay statically
//   indexed.  Reductions are xor butterflies: every lane gets the same value, and repeated calls are bit-identical.
constexpr int kEnetThreads = 256;
constexpr double kEnetConstCol = 1e-12;
constexpr double kF64Resolution = 1e-15;     // np.finfo(np.float64).resolution

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// gap_enet_gram: formulation A (l1 > 0), B (l1 == 0 < l2) or the squared OLS gradient (both 0); xta = X^T R - l2 w (X^T R
// without an L1 term) per owned feature, *dual_norm as sklearn's dual_norm_XtA.  Features >= d hold zeros throughout.
__device__ __forceinline__ double enet_gap(const double (&w)[4], const double (&qw)[4], const double (&q)[4], int d,
                                           int lane, double l1, double l2, double y_norm2, bool positive,
                                           double (&xta)[4], double* dual_norm) {
  double ww = 0.0, qdw = 0.0, wqw = 0.0, wl1 = 0.0, dn = l1 == 0.0 ? 0.0 : -INFINITY;
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const bool live = lane + 32 * u < d;
    ww = fma(w[u], w[u], ww);
    qdw = fma(w[u], q[u], qdw);
    wqw = fma(w[u], qw[u], wqw);
    wl1 += fabs(w[u]);
    if (l1 == 0.0) {
      xta[u] = q[u] - qw[u];
      dn = fma(xta[u], xta[u], dn);
    } else {
      xta[u] = q[u] - qw[u] - l2 * w[u];
      if (live) dn = fmax(dn, positive ? xta[u] : fabs(xta[u]));
    }
  }
  qdw = warp_sum(qdw);
  wqw = warp_sum(wqw);
  ww = l2 > 0.0 ? warp_sum(ww) : 0.0;
  const double r_norm2 = y_norm2 + wqw - 2.0 * qdw;
  const double ry = y_norm2 - qdw;
  if (l1 == 0.0) {
    dn = warp_sum(dn);
    *dual_norm = dn;
    if (l2 == 0.0) return dn;
    return r_norm2 + 0.5 * l2 * ww - ry + 1.0 / (2.0 * l2) * dn;
  }
  dn = warp_max(dn);
  wl1 = warp_sum(wl1);
  *dual_norm = dn;
  const double primal = 0.5 * (r_norm2 + l2 * ww) + l1 * wl1;
  const double scale = dn > l1 ? l1 / dn : 1.0;
  const double dual = -0.5 * (scale * scale) * (r_norm2 + l2 * ww) + scale * ry;
  return primal - dual;
}

// The statistic a CTA of solve_enet_kernel reads: S itself (folds == nullptr), or the sum of the fold statistics other
// than fold `skip` (skip < 0: all of them), added in fold order from 0 -- the additions fold_sum_kernel makes for S.
struct FoldStat {
  const double* S;
  const double* folds;
  int n_folds, skip, stride;
  __device__ __forceinline__ double operator()(int i) const {
    if (folds == nullptr) return __ldcg(S + i);
    double t = 0.0;
    for (int j = 0; j < n_folds; ++j)
      if (j != skip) t += __ldcg(folds + (size_t)j * stride + i);
    return t;
  }
};

// Warp 0 after a build of Q / r from S: constant columns get their Q row and column and their q entry zeroed (the
// build's last barrier preceded this); lane l gets the live bits, q and Q_jj of features l + 32 u.
__device__ __forceinline__ void enet_columns(const FoldStat& S, double* Q, double* r, int d, int lane,
                                             unsigned int (&live)[4], double (&q)[4], double (&qjj)[4]) {
  const int pitch = d + 1, dp = d + 2;
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int f = lane + 32 * u;
    const bool ok = f < d && Q[f * pitch + f] > kEnetConstCol * S(f * dp + f);
    const bool dead = f < d && !ok;
    live[u] = __ballot_sync(0xffffffffu, ok);
    unsigned int m = __ballot_sync(0xffffffffu, dead);
    while (m) {
      const int j = __ffs(m) - 1 + 32 * u;
      m &= m - 1;
#pragma unroll
      for (int v = 0; v < 4; ++v) {
        const int g = lane + 32 * v;
        if (g < d) { Q[j * pitch + g] = 0.0; Q[g * pitch + j] = 0.0; }
      }
      if (lane == 0) r[j] = 0.0;
    }
  }
  __syncwarp();
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int f = lane + 32 * u;
    q[u] = f < d ? r[f] : 0.0;
    qjj[u] = f < d ? Q[f * pitch + f] : 0.0;
  }
}

// sklearn's _alpha_grid: alpha_max = max |q| (max q with positive) / (n l1_ratio), then alpha i of
// geomspace(alpha_max, alpha_max eps, n_alphas), or a constant grid at the fp64 resolution
__device__ __forceinline__ double enet_alpha_max(const double (&q)[4], double n, double l1_ratio, bool positive) {
  double mx = 0.0;
#pragma unroll
  for (int u = 0; u < 4; ++u) mx = fmax(mx, positive ? q[u] : fabs(q[u]));
  return warp_max(mx) / (n * l1_ratio);
}
__device__ __forceinline__ double enet_grid_alpha(int i, double amax, double eps, int n_alphas) {
  const double amin = amax * eps;
  const double ls = log10(amax), step = n_alphas > 1 ? (log10(amin) - ls) / (double)(n_alphas - 1) : 0.0;
  double v = exp10(__dadd_rn(__dmul_rn((double)i, step), ls));
  if (i == 0) v = amax;
  if (i == n_alphas - 1 && i > 0) v = amin;
  return amax <= kF64Resolution ? kF64Resolution : v;
}

// One CTA per (l1_ratio l, fold k): blockIdx.x = l n_folds + k.  b2_solve_enet_path is the case n_folds = 1 without
// folds (the path of S).  Cross-validation (a.folds): the grid comes from the summed statistic, built and screened as
// the path's own; the path runs on T_k = the sum of the other folds; then all warps form the held-out error of every
// alpha from S_k (DESIGN.md section 8).
__global__ void __launch_bounds__(kEnetThreads, 1)
solve_enet_kernel(const double* __restrict__ S, int d, EnetArgs a) {
  extern __shared__ double sm[];
  const int pitch = d + 1, dp = d + 2;
  double* Q = sm;                          // d x d, pitch d + 1; row d = q
  double* r = Q + d * pitch;
  double* mean = Q + (d + 1) * pitch;
  double* wsh = mean + d;                  // [kMaxD] w at the start of an alpha (for Q w)
  double* misc = wsh + kMaxD;              // [0] ybar
  const int l = blockIdx.x / a.n_folds, k = blockIdx.x - l * a.n_folds;
  const double l1_ratio = a.l1_ratios != nullptr ? a.l1_ratios[l] : a.l1_ratio;
  const bool positive = a.positive != 0;
  const int lane = threadIdx.x & 31;
  const size_t A = (size_t)a.n_alphas;
  double* coefs = a.coefs + blockIdx.x * A * d;
  double* intercepts = a.intercepts + blockIdx.x * A;
  double amax = 0.0;
  if (a.folds != nullptr) {
    const FoldStat all{S, a.folds, a.n_folds, -1, dp * dp};
    build_normal_equations_of(all, d, 0.0, a.fit_intercept, Q, r, mean, &misc[0]);
    if (threadIdx.x < 32) {
      unsigned int live[4];
      double q[4], qjj[4];
      enet_columns(all, Q, r, d, lane, live, q, qjj);
      amax = enet_alpha_max(q, all(d * dp + d), l1_ratio, positive);
    }
    __syncthreads();
  }
  const FoldStat st{S, a.folds, a.n_folds, k, dp * dp};
  build_normal_equations_of(st, d, 0.0, a.fit_intercept, Q, r, mean, &misc[0]);
  if (threadIdx.x < 32) {                  // one warp from here to the end of the path: __syncwarp only
    const double n = st(d * dp + d);
    const double ybar = misc[0];
    const double y_norm2 = st((d + 1) * dp + d + 1) - n * ybar * ybar;
    unsigned int live[4];
    double w[4], qw[4], q[4], qjj[4], rinv[4], xta[4];
    enet_columns(st, Q, r, d, lane, live, q, qjj);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const bool ok = (live[u] >> lane) & 1u;
      w[u] = (ok && a.coef_init != nullptr) ? a.coef_init[lane + 32 * u] : 0.0;
    }
    if (a.folds == nullptr) amax = enet_alpha_max(q, n, l1_ratio, positive);
    if (a.grid && k == 0)
      for (int i = lane; i < a.n_alphas; i += 32) a.alphas[l * A + i] = enet_grid_alpha(i, amax, a.eps, a.n_alphas);

    const double tol_abs = a.tol * y_norm2;
    if (lane == 0) a.tol_out[blockIdx.x] = tol_abs / n;
    for (int ia = 0; ia < a.n_alphas; ++ia) {
      const double alpha = a.grid ? enet_grid_alpha(ia, amax, a.eps, a.n_alphas) : a.alphas[ia];
      const double l1 = alpha * l1_ratio * n, l2 = alpha * (1.0 - l1_ratio) * n;
      // Qw = Q w from scratch (as sklearn's np.dot at every alpha), Q read by columns: lane-consecutive addresses
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (lane + 32 * u < d) wsh[lane + 32 * u] = w[u];
        rinv[u] = qjj[u] > 0.0 ? 1.0 / (qjj[u] + l2) : 0.0;
        qw[u] = 0.0;
      }
      __syncwarp();
      for (int j = 0; j < d; ++j) {
        const double wj = wsh[j];
#pragma unroll
        for (int u = 0; u < 4; ++u)
          if (lane + 32 * u < d) qw[u] = fma(Q[j * pitch + lane + 32 * u], wj, qw[u]);
      }
      double dn;
      double gap = enet_gap(w, qw, q, d, lane, l1, l2, y_norm2, positive, xta, &dn);
      int iters = 0;
      if (!(gap >= 0.0 && gap <= tol_abs)) {
        const bool screening = l1 > 0.0;
        unsigned int act[4];
        // gap-safe screening (sklearn: Fercoq et al. eq. 11) over the candidates `cand`: kept features form the active
        // set, the others leave it for good, their w (if any) taken out of Qw in feature order
        auto screen = [&](const unsigned int (&cand)[4]) {
          const double radius = sqrt(2.0 * fabs(gap)) / l1;
          const double theta_scale = fmax(l1, dn);
          unsigned int drop[4];
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const bool c = (cand[u] >> lane) & 1u;
            const bool keep = c && qjj[u] != 0.0 && (1.0 - fabs(xta[u] / theta_scale)) / sqrt(qjj[u] + l2) <= radius;
            act[u] = __ballot_sync(0xffffffffu, keep);
            drop[u] = __ballot_sync(0xffffffffu, c && !keep && w[u] != 0.0);
          }
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            unsigned int m = drop[u];
            while (m) {
              const int j = __ffs(m) - 1;
              m &= m - 1;
              const double wj = __shfl_sync(0xffffffffu, w[u], j);
              if (lane == j) w[u] = 0.0;
              const double* row = Q + (j + 32 * u) * pitch;
#pragma unroll
              for (int v = 0; v < 4; ++v)
                if (lane + 32 * v < d) qw[v] = fma(-wj, row[lane + 32 * v], qw[v]);
            }
          }
        };
        if (screening) {
          unsigned int all[4];
#pragma unroll
          for (int u = 0; u < 4; ++u) all[u] = __ballot_sync(0xffffffffu, lane + 32 * u < d);
          screen(all);
        } else {
#pragma unroll
          for (int u = 0; u < 4; ++u) act[u] = live[u];
        }
        iters = a.max_iter;
        for (int it = 0; it < a.max_iter; ++it) {
          double dw_max = 0.0, w_max = 0.0;
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            unsigned int m = act[u];
            while (m) {
              const int j = __ffs(m) - 1;
              m &= m - 1;
              const double* row = Q + (j + 32 * u) * pitch;
              double rv[4];                                  // row j: its loads do not wait for the step
#pragma unroll
              for (int v = 0; v < 4; ++v) rv[v] = lane + 32 * v < d ? row[lane + 32 * v] : 0.0;
              // Branch-free: every lane evaluates the update of its own feature lane + 32 u and the shuffle takes lane
              // j's.  The chain per coordinate is t -> soft threshold -> step -> shuffle -> the owner's Qw FMA.  A zero
              // step adds an exact zero to Qw (sklearn skips it; the value is the same).
              const double wj = w[u];
              const double t = fma(wj, qjj[u], q[u]) - qw[u];
              const double mag = fmax(fabs(t) - l1, 0.0) * rinv[u];
              const double nw = (positive && t < 0.0) ? 0.0 : (t > 0.0 ? mag : (t < 0.0 ? -mag : 0.0));
              const double delta = __shfl_sync(0xffffffffu, nw - wj, j);
              const bool own = lane == j;
              w[u] = own ? nw : wj;
              dw_max = own ? fmax(dw_max, fabs(delta)) : dw_max;
              w_max = own ? fmax(w_max, fabs(nw)) : w_max;
#pragma unroll
              for (int v = 0; v < 4; ++v) qw[v] = fma(delta, rv[v], qw[v]);
            }
          }
          dw_max = warp_max(dw_max);
          w_max = warp_max(w_max);
          if (w_max == 0.0 || dw_max / w_max <= a.tol || it == a.max_iter - 1) {
            gap = enet_gap(w, qw, q, d, lane, l1, l2, y_norm2, positive, xta, &dn);
            if (gap <= tol_abs) {
              iters = it + 1;
              break;
            }
            if (screening) {
              const unsigned int cand[4] = {act[0], act[1], act[2], act[3]};
              screen(cand);
            }
          }
        }
      }
      double part = 0.0;
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int f = lane + 32 * u;
        if (f < d) {
          coefs[(size_t)ia * d + f] = w[u];
          part = fma(mean[f], w[u], part);
        }
      }
      part = warp_sum(part);
      if (lane == 0) {
        intercepts[ia] = ybar - part;
        a.gaps[blockIdx.x * A + ia] = gap / n;
        a.iters[blockIdx.x * A + ia] = (double)iters;
      }
    }
  }
  if (a.folds == nullptr) return;
  __syncthreads();                         // the path's coefficients and intercepts are in global memory; Q is free
  // Held-out error of every alpha from the fold's own statistic S_k: C = the centred second moments of [x y] (y last,
  // symmetric, pitch d + 1 in Q's place), mu and vbar its means.  mse = (vbar - b - mu.w)^2 + w~^T C w~ / n_k with
  // w~ = [w; -1], the quadratic term clamped at 0.  Warp v takes alphas v, v + 8, ...; lane l rows l + 32 u of C w~.
  const double* Sk = a.folds + (size_t)k * dp * dp;
  const double nk = __ldcg(Sk + d * dp + d);
  double* C = Q;
  double* mu = wsh;                        // [d] means of x; misc[1] the mean of y
  for (int i = threadIdx.x; i <= d; i += blockDim.x) {
    const double m = __ldcg(Sk + (i < d ? i : d + 1) * dp + d) / nk;
    if (i < d) mu[i] = m;
    else misc[1] = m;
  }
  __syncthreads();
  for (int t = threadIdx.x; t < pitch * pitch; t += blockDim.x) {
    const int i = t / pitch, j = t - i * pitch;
    const double mi = i < d ? mu[i] : misc[1], mj = j < d ? mu[j] : misc[1];
    C[t] = __ldcg(Sk + (i < d ? i : d + 1) * dp + (j < d ? j : d + 1)) - nk * mi * mj;
  }
  __syncthreads();
  const double vbar = misc[1];
  for (int ia = threadIdx.x >> 5; ia < a.n_alphas; ia += kEnetThreads / 32) {
    const double* w = coefs + (size_t)ia * d;
    double cw[5] = {0.0, 0.0, 0.0, 0.0, 0.0};   // (C w~)_i, i = lane + 32 u <= d
    for (int j = 0; j <= d; ++j) {
      const double wj = j < d ? w[j] : -1.0;
#pragma unroll
      for (int u = 0; u < 5; ++u)
        if (lane + 32 * u <= d) cw[u] = fma(C[j * pitch + lane + 32 * u], wj, cw[u]);
    }
    double quad = 0.0, mw = 0.0;
#pragma unroll
    for (int u = 0; u < 5; ++u) {
      const int i = lane + 32 * u;
      if (i < d) {
        quad = fma(w[i], cw[u], quad);
        mw = fma(mu[i], w[i], mw);
      } else if (i == d) {
        quad -= cw[u];
      }
    }
    quad = warp_sum(quad);
    mw = warp_sum(mw);
    if (lane == 0) {
      const double res = vbar - intercepts[ia] - mw;
      a.mse[((size_t)l * A + ia) * a.n_folds + k] = res * res + fmax(quad, 0.0) / nk;
    }
  }
}

size_t enet_smem_bytes(int d) { return sizeof(double) * ((size_t)(d + 1) * (d + 1) + d + kMaxD + 8); }

// ---- BayesianRidge and ARDRegression: evidence maximisation on the centred Gram (b2_solve_bayes_ridge, b2_solve_ard) --
// Both restate scikit-learn 1.9's fit loops (sklearn/linear_model/_bayes.py) on the fp64 statistic; DESIGN.md section 9.
// The residual sum of squares both need comes from the anchor (b2_residual_moments at w0: g0 = sum (x - m) e, s0 = sum e,
// sse0 = sum e^2), exactly: sse(w) = sse0 - s0^2 / n - 2 D.g0 + D^T A D with D = w - w0; without an anchor from S alone,
// sse(w) = ||yc||^2 - 2 w.r + w^T A w.  Every reduction is a warp butterfly, then the warps in order, so repeated calls are
// bit-identical.
constexpr int kByThreads = 512;
constexpr double kF64Eps = 2.220446049250313e-16;    // np.finfo(np.float64).eps
constexpr double kLog2Pi = 1.8378770664093453;       // log(2 pi)

// the sum of every thread's v, in a fixed order, returned to every thread; red: blockDim.x / 32 doubles
__device__ __forceinline__ double block_sum(double v, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += red[w];
  __syncthreads();
  return s;
}

// row . x over the first d entries with 4 threads per row (thread = 4 row + part); every thread of a warp must call it
// (a row past the matrix passes d = 0).  The four partial sums are combined by a fixed butterfly.
__device__ __forceinline__ double row_dot4(const double* __restrict__ rowp, const double* __restrict__ x, int d, int part) {
  double v = 0.0;
  for (int j = part; j < d; j += 4) v = fma(rowp[j], x[j], v);
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  v += __shfl_xor_sync(0xffffffffu, v, 2);
  return v;
}

// n, ybar (0 without an intercept), ||yc||^2 (||y||^2 without an intercept) and y.var() (always about the mean) from S
struct YStats {
  double n, ybar, yy, y_var;
};
__device__ __forceinline__ YStats y_stats(const double* __restrict__ S, int d, int fit_intercept) {
  const int dp = d + 2;
  const double n = S[d * dp + d], sy = S[d * dp + d + 1], syy = S[(d + 1) * dp + d + 1];
  const double inv_n = n > 0.0 ? 1.0 / n : 0.0;
  YStats t;
  t.n = n;
  t.ybar = fit_intercept ? sy * inv_n : 0.0;
  t.yy = fit_intercept ? syy - n * t.ybar * t.ybar : syy;
  t.y_var = fmax(syy * inv_n - (sy * inv_n) * (sy * inv_n), 0.0);
  return t;
}

size_t bayes_smem_bytes(int d) { return sizeof(double) * ((size_t)d * (d + 1) + 8 * kMaxD + 32); }

// BayesianRidge.fit in the eigenbasis A = Q diag(lam) Q^T of solve_eigh_kernel (ctx->loo): w~ = c / (lam + lambda_ /
// alpha_), coef = Q w~ every iteration (the stopping test sum |coef_old - coef| < tol is in the original basis),
// gamma = sum alpha_ lam / (lambda_ + alpha_ lam), then lambda_ and alpha_ in scikit-learn's order.  With an anchor
// D~ = w~ - Q^T w0 and g~0 = Q^T g0 are formed once, so sse = sse0 - s0^2 / n + sum lam D~^2 - 2 D~.g~0; without one
// sse = ||yc||^2 - sum c^2 (lam + 2 s) / (lam + s)^2, s = lambda_ / alpha_.  logdet runs over all d eigenvalues, which is
// scikit-learn's n <= d branch as well (the eigenvalues past rank n are 0).  Finally sigma = Q diag(1 / (alpha_ lam +
// lambda_)) Q^T, its upper triangle mirrored.
__global__ void __launch_bounds__(kByThreads, 1)
bayes_ridge_kernel(const double* __restrict__ S, int d, const double* __restrict__ loo, const BayesArgs a) {
  extern __shared__ double sm[];
  const int pitch = d + 1;
  double* Qs = sm;                    // Q[i][k], pitch d + 1
  double* lam = Qs + d * pitch;
  double* c = lam + kMaxD;            // Q^T r
  double* wt = c + kMaxD;             // w~
  double* coef = wt + kMaxD;
  double* coef_old = coef + kMaxD;
  double* w0t = coef_old + kMaxD;     // Q^T w0
  double* g0t = w0t + kMaxD;          // Q^T g0
  double* inv = g0t + kMaxD;          // 1 / (alpha_ lam + lambda_)
  double* red = inv + kMaxD;          // [32]
  const int tid = threadIdx.x, row = tid >> 2, part = tid & 3;
  for (int t = tid; t < d * d; t += blockDim.x) {
    const int i = t / d, k = t - i * d;
    Qs[i * pitch + k] = loo[kLooQ + i * kMaxD + k];
  }
  for (int k = tid; k < d; k += blockDim.x) {
    lam[k] = loo[kLooLam + k];
    c[k] = loo[kLooC + k];
  }
  const YStats ys = y_stats(S, d, a.fit_intercept);
  const double n = ys.n;
  const bool anchored = a.anchor != nullptr;
  double sse_base = ys.yy;
  __syncthreads();
  if (anchored) {
    for (int k = tid; k < d; k += blockDim.x) {
      double w = 0.0, g = 0.0;
      for (int i = 0; i < d; ++i) {
        w = fma(Qs[i * pitch + k], a.anchor[i], w);
        g = fma(Qs[i * pitch + k], a.anchor[kMaxD + i], g);
      }
      w0t[k] = w;
      g0t[k] = g;
    }
    const double s0 = a.anchor[2 * kMaxD], sse0 = a.anchor[2 * kMaxD + 1];
    sse_base = sse0 - (a.fit_intercept && n > 0.0 ? s0 * s0 / n : 0.0);
    __syncthreads();
  }
  double alpha = isnan(a.alpha_init) ? 1.0 / (ys.y_var + kF64Eps) : a.alpha_init;
  double lmb = isnan(a.lambda_init) ? 1.0 : a.lambda_init;
  // coef and sse at (alpha, lmb)
  auto update_coef = [&]() -> double {
    const double s = lmb / alpha;
    double term = 0.0;
    if (tid < d) {
      const double q = lam[tid] + s, w = c[tid] / q;
      wt[tid] = w;
      if (anchored) {
        const double dt = w - w0t[tid];
        term = fma(lam[tid] * dt, dt, -2.0 * dt * g0t[tid]);
      } else {
        term = -(c[tid] * c[tid]) * (lam[tid] + 2.0 * s) / (q * q);
      }
    }
    const double sse = sse_base + block_sum(term, red);   // its barriers publish wt
    const double v = row_dot4(Qs + (row < d ? row : 0) * pitch, wt, row < d ? d : 0, part);
    if (row < d && part == 0) coef[row] = v;
    __syncthreads();
    return sse;
  };
  auto score = [&](double sse) -> double {   // _log_marginal_likelihood
    double ld = 0.0, cs = 0.0;
    if (tid < d) {
      ld = log(lmb + alpha * lam[tid]);
      cs = coef[tid] * coef[tid];
    }
    const double logdet = -block_sum(ld, red);
    const double csq = block_sum(cs, red);
    double s = a.l1 * log(lmb) - a.l2 * lmb;
    s += a.a1 * log(alpha) - a.a2 * alpha;
    s += 0.5 * (d * log(lmb) + n * log(alpha) - alpha * sse - lmb * csq + logdet - n * kLog2Pi);
    return s;
  };
  int iter = 0;
  for (; iter < a.max_iter; ++iter) {
    const double sse = update_coef();
    if (a.compute_score) {
      const double s = score(sse);
      if (tid == 0) a.scores[iter] = s;
    }
    double gl = 0.0, cs = 0.0;
    if (tid < d) {
      gl = alpha * lam[tid] / (lmb + alpha * lam[tid]);
      cs = coef[tid] * coef[tid];
    }
    const double gamma = block_sum(gl, red);
    const double csq = block_sum(cs, red);
    lmb = (gamma + 2.0 * a.l1) / (csq + 2.0 * a.l2);
    alpha = (n - gamma + 2.0 * a.a1) / (sse + 2.0 * a.a2);
    if (iter != 0 && block_sum(tid < d ? fabs(coef_old[tid] - coef[tid]) : 0.0, red) < a.tol) break;
    if (tid < d) coef_old[tid] = coef[tid];
  }
  const int n_iter = iter < a.max_iter ? iter + 1 : a.max_iter;
  const double sse = update_coef();
  if (a.compute_score) {
    const double s = score(sse);
    if (tid == 0) a.scores[n_iter] = s;
  }
  for (int k = tid; k < d; k += blockDim.x) inv[k] = 1.0 / (alpha * lam[k] + lmb);
  const double mc = block_sum(tid < d ? loo[kLooMean + tid] * coef[tid] : 0.0, red);
  for (int t = tid; t < d * d; t += blockDim.x) {
    const int i = t / d, j = t - i * d;
    if (i > j) continue;
    double v = 0.0;
    for (int k = 0; k < d; ++k) v = fma(Qs[i * pitch + k] * inv[k], Qs[j * pitch + k], v);
    a.out[kBySigma + i * d + j] = v;
    a.out[kBySigma + j * d + i] = v;
  }
  if (tid < d) a.out[kByCoef + tid] = coef[tid];
  if (tid == 0) {
    a.out[kByMisc + 0] = a.fit_intercept ? ys.ybar - mc : 0.0;
    a.out[kByMisc + 1] = alpha;
    a.out[kByMisc + 2] = lmb;
    a.out[kByMisc + 3] = n_iter;
    a.out[kByMisc + 4] = 0.0;
  }
}

size_t ard_smem_bytes(int d) { return sizeof(double) * ((size_t)d * (d + 1) + 8 * kMaxD + 32 + 8); }

// ARDRegression.fit.  Per iteration: M = diag(lambda) + alpha A on the kept set, with a unit row and column for every
// pruned feature, so pruned features decouple and the kept block of M^-1 is scikit-learn's sigma_; M^-1 by the sweep
// operator in place (M becomes -M^-1; the pivots are the LDL^T pivots, so log det M = sum log pivot); coef_K = alpha
// sigma r_K; sse from the anchor (with A D); gamma = 1 - lambda sigma_jj, lambda_K, alpha; then the prune (keep = lambda <
// threshold_lambda), the score (fast_logdet(sigma) = -log det M) and the stopping test, in scikit-learn's order: sse uses
// the coefficients before the prune, the score and the test those after it.  A non-positive pivot stops the kernel with
// info = its index + 1.  A (the centred Gram) lives in global memory beside the outputs: with M it would not fit in
// shared memory at d = 128, and two matrix-vector reads of it per iteration come from L2.
__global__ void __launch_bounds__(kByThreads, 1)
ard_kernel(const double* __restrict__ S, int d, const BayesArgs a) {
  extern __shared__ double sm[];
  const int pitch = d + 1;
  double* M = sm;
  double* r = M + d * pitch;
  double* mean = r + kMaxD;
  double* lmb = mean + kMaxD;
  double* coef = lmb + kMaxD;
  double* coef_old = coef + kMaxD;
  double* keep = coef_old + kMaxD;    // 1: kept
  double* col = keep + kMaxD;         // the pivot column of a sweep step
  double* dlt = col + kMaxD;          // coef - w0
  double* red = dlt + kMaxD;          // [32]
  double* misc = red + 32;            // [0] ybar, [1] info
  double* A = a.A;
  const int tid = threadIdx.x, row = tid >> 2, part = tid & 3;
  if (tid == 0) misc[1] = 0.0;
  build_normal_equations(S, d, 0.0, a.fit_intercept, M, r, mean, &misc[0]);
  for (int t = tid; t < d * d; t += blockDim.x) {
    const int i = t / d, j = t - i * d;
    A[t] = M[i * pitch + j];
  }
  for (int j = tid; j < d; j += blockDim.x) {
    lmb[j] = 1.0;
    coef[j] = 0.0;
    keep[j] = 1.0;
  }
  const YStats ys = y_stats(S, d, a.fit_intercept);
  const double n = ys.n;
  const bool anchored = a.anchor != nullptr;
  const double sse_base = anchored ? a.anchor[2 * kMaxD + 1] -
                                         (a.fit_intercept && n > 0.0 ? a.anchor[2 * kMaxD] * a.anchor[2 * kMaxD] / n : 0.0)
                                   : ys.yy;
  __syncthreads();
  double alpha = 1.0 / (ys.y_var + kF64Eps);
  // M -> -M^-1; returns log det M, NaN after a non-positive pivot.  Entry (i, j) becomes M_ij - (M_ik M_kj) / p, which
  // keeps M exactly symmetric.
  auto sweep = [&]() -> double {
    double logdet = 0.0;
    for (int k = 0; k < d; ++k) {
      for (int i = tid; i < d; i += blockDim.x) col[i] = M[i * pitch + k];
      __syncthreads();
      const double p = col[k];
      if (!(p > 0.0)) {                           // the same p in every thread: a uniform exit
        if (tid == 0) misc[1] = k + 1;
        return NAN;
      }
      const double rp = 1.0 / p;
      logdet += log(p);
      for (int t = tid; t < d * d; t += blockDim.x) {
        const int i = t / d, j = t - i * d;
        double v;
        if (i == k) v = j == k ? -rp : col[j] * rp;
        else if (j == k) v = col[i] * rp;
        else v = M[i * pitch + j] - (col[i] * col[j]) * rp;
        M[i * pitch + j] = v;
      }
      __syncthreads();
    }
    return logdet;
  };
  // M of the current (alpha, lambda, keep), sigma, coef_K = alpha sigma r_K
  auto solve = [&]() -> double {
    for (int t = tid; t < d * d; t += blockDim.x) {
      const int i = t / d, j = t - i * d;
      const bool kk = keep[i] != 0.0 && keep[j] != 0.0;
      M[i * pitch + j] = kk ? fma(alpha, A[t], i == j ? lmb[i] : 0.0) : (i == j ? 1.0 : 0.0);
    }
    for (int j = tid; j < d; j += blockDim.x) dlt[j] = keep[j] != 0.0 ? r[j] : 0.0;
    __syncthreads();
    const double ld = sweep();
    if (isnan(ld)) return ld;
    const double v = row_dot4(M + (row < d ? row : 0) * pitch, dlt, row < d ? d : 0, part);
    if (row < d && part == 0 && keep[row] != 0.0) coef[row] = -alpha * v;
    __syncthreads();
    return ld;
  };
  auto sse_of = [&]() -> double {
    if (tid < d) dlt[tid] = coef[tid] - (anchored ? a.anchor[tid] : 0.0);
    __syncthreads();
    const double v = row_dot4(A + (row < d ? row : 0) * d, dlt, row < d ? d : 0, part);
    double term = 0.0;
    if (row < d && part == 0) term = dlt[row] * (v - 2.0 * (anchored ? a.anchor[kMaxD + row] : r[row]));
    return sse_base + block_sum(term, red);
  };
  double nkeep = d;
  bool singular = false;
  int iter = 0;
  for (; iter < a.max_iter; ++iter) {
    const double ld = solve();
    if (isnan(ld)) {
      singular = true;
      break;
    }
    const double sse = sse_of();
    double g = 0.0;
    if (tid < d && keep[tid] != 0.0) {
      g = 1.0 + lmb[tid] * M[tid * pitch + tid];   // 1 - lambda_j sigma_jj
      lmb[tid] = (g + 2.0 * a.l1) / (coef[tid] * coef[tid] + 2.0 * a.l2);
    }
    alpha = (n - block_sum(g, red) + 2.0 * a.a1) / (sse + 2.0 * a.a2);
    double kept = 0.0;
    if (tid < d) {
      kept = lmb[tid] < a.threshold_lambda ? 1.0 : 0.0;
      keep[tid] = kept;
      if (kept == 0.0) coef[tid] = 0.0;
    }
    nkeep = block_sum(kept, red);
    if (a.compute_score) {
      double t1 = 0.0, t2 = 0.0, t3 = 0.0;
      if (tid < d) {
        t1 = a.l1 * log(lmb[tid]) - a.l2 * lmb[tid];
        t2 = log(lmb[tid]);
        t3 = lmb[tid] * coef[tid] * coef[tid];
      }
      double s = block_sum(t1, red);
      const double slog = block_sum(t2, red), sq = block_sum(t3, red);
      s += a.a1 * log(alpha) - a.a2 * alpha;
      s += 0.5 * (-ld + n * log(alpha) + slog);
      s -= 0.5 * (alpha * sse + sq);
      if (tid == 0) a.scores[iter] = s;
    }
    if (iter > 0 && block_sum(tid < d ? fabs(coef_old[tid] - coef[tid]) : 0.0, red) < a.tol) break;
    if (tid < d) coef_old[tid] = coef[tid];
    if (nkeep == 0.0) break;
  }
  const int n_iter = iter < a.max_iter ? iter + 1 : a.max_iter;
  if (!singular && nkeep > 0.0 && isnan(solve())) singular = true;
  const double mc = block_sum(tid < d ? mean[tid] * coef[tid] : 0.0, red);
  for (int t = tid; t < d * d; t += blockDim.x) {
    const int i = t / d, j = t - i * d;
    a.out[kBySigma + t] = !singular && nkeep > 0.0 && keep[i] != 0.0 && keep[j] != 0.0 ? -M[i * pitch + j] : 0.0;
  }
  if (tid < d) {
    a.out[kByCoef + tid] = coef[tid];
    a.out[kByLambda + tid] = lmb[tid];
  }
  if (tid == 0) {
    a.out[kByMisc + 0] = a.fit_intercept ? misc[0] - mc : 0.0;
    a.out[kByMisc + 1] = alpha;
    a.out[kByMisc + 3] = n_iter;
    a.out[kByMisc + 4] = misc[1];
  }
}

// ---- the ridge classifier's solve (b2_solve_classes; DESIGN.md section 12) ---------------------------------------------
// (Xc^T Xc + alpha I) W^T = Xc^T Yc for the T = n_classes targets (1 with two classes: the second class is the positive
// one) of LabelBinarizer(pos_label=1, neg_label=-1).  From the class sums s_k = sum_{y = k} (x - c) and counts n_k of
// the kept rows (any centre c, every kept row of some class), with s = sum_k s_k and n the rows of S:
//   Xc^T Yc[:, k] = sum (x - c)(y_k - ybar_k) = 2 (s_k - (n_k / n) s)   (2 s_k - s without an intercept, c = 0)
//   b_k = ybar_k - mean.w_k,  ybar_k = 2 n_k / n - 1.
// A is build_normal_equations'; the T right-hand sides ride as extra rows of [A ; Rhs^T] through an unblocked
// right-looking LDL^T (the pivot rule of solve_cholesky_kernel: a pivot <= 1e-12 of the largest diagonal entry refuses the
// system), which leaves D^-1 M^-1 r_t in row d + t; then M^T w_t = that row, one warp per target.
constexpr int kClsThreads = 512;
size_t solve_classes_smem_bytes(int d, int n_targets) {
  return sizeof(double) * ((size_t)(d + n_targets) * (d + 1) + 3 * kMaxD + kMaxClasses + 16);
}

__global__ void __launch_bounds__(kClsThreads, 1)
solve_classes_kernel(double* S, int d, double alpha, int fit_intercept, int n_classes, double* __restrict__ cls) {
  extern __shared__ double sm[];
  const int T = n_classes == 2 ? 1 : n_classes, pitch = d + 1, rows = d + T;
  double* A = sm;                          // rows 0..d-1 = A, row d + t = the right-hand side of target t
  double* mean = A + rows * pitch;         // [kMaxD]
  double* tot = mean + kMaxD;              // [kMaxD] s = sum_k s_k
  double* col = tot + kMaxD;               // [kMaxD + kMaxClasses] column k of the current step
  double* misc = col + kMaxD + kMaxClasses;   // [0] ybar of S (unused), [1] the largest diagonal entry
  const double* sums = cls + kClsSums;     // [K][d + 1]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
  build_normal_equations(S, d, alpha, fit_intercept, A, A + d * pitch, mean, &misc[0]);
  const double n = __ldcg(S + d * (d + 2) + d);
  if (tid < d) {
    double s = 0.0;
    for (int k = 0; k < n_classes; ++k) s += sums[k * (d + 1) + tid];
    tot[tid] = s;
  }
  __syncthreads();
  for (int t = tid; t < T * d; t += blockDim.x) {
    const int tt = t / d, j = t - tt * d, k = T == 1 ? 1 : tt;
    const double sk = sums[k * (d + 1) + j], nk = sums[k * (d + 1) + d];
    A[(d + tt) * pitch + j] = fit_intercept ? 2.0 * (sk - (nk / n) * tot[j]) : 2.0 * sk - tot[j];
  }
  if (warp == 0) {
    double mx = 0.0;
    for (int i = lane; i < d; i += 32) mx = fmax(mx, A[i * pitch + i]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (lane == 0) misc[1] = mx;
  }
  __syncthreads();
  const double tiny = misc[1] * 1e-12;
  int info = 0;
  for (int k = 0; k < d; ++k) {
    const double piv = A[k * pitch + k];
    if (!(piv > tiny)) { info = k + 1; break; }   // block-uniform
    const double rc = 1.0 / piv;
    for (int i = k + 1 + tid; i < rows; i += blockDim.x) col[i] = A[i * pitch + k];
    __syncthreads();
    // a_ij -= u_ik u_jk / D_k for k < j <= i (every j > k in the right-hand sides); m_ik = u_ik / D_k; warp per row
    for (int i = k + 1 + warp; i < rows; i += nwarps) {
      const double f = col[i] * rc;
      const int jend = i < d ? i : d - 1;
      for (int j = k + 1 + lane; j <= jend; j += 32) A[i * pitch + j] = fma(-f, col[j], A[i * pitch + j]);
      if (lane == 0) A[i * pitch + k] = f;
    }
    __syncthreads();
  }
  // M^T w = z per target, from the bottom: w_i is final once every m > i has been subtracted
  for (int t = warp; t < T; t += nwarps) {
    double* z = A + (d + t) * pitch;
    if (info == 0) {
      for (int i = d - 1; i > 0; --i) {
        const double wi = z[i];
        for (int m = lane; m < i; m += 32) z[m] = fma(-A[i * pitch + m], wi, z[m]);
        __syncwarp();
      }
    }
    double part = 0.0;
    for (int j = lane; j < d; j += 32) {
      const double w = info == 0 ? z[j] : 0.0;
      cls[kClsCoef + t * kMaxD + j] = w;
      part = fma(mean[j], w, part);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
    if (lane == 0) {
      const int k = T == 1 ? 1 : t;
      const double ybar = fit_intercept ? 2.0 * sums[k * (d + 1) + d] / n - 1.0 : 0.0;
      cls[kClsIntercept + t] = info == 0 ? ybar - part : 0.0;
    }
  }
  if (tid == 0) cls[kClsInfo] = (double)info;
}

size_t solve_smem_bytes(int d) {
  // Cholesky: A, mean, invd, misc, U panel; eigenvalue kernel: A, r, mean, misc, (v, w) x 2, pv, dd, ee2, lam
  const size_t chol = (size_t)(d + 1) * (d + 1) + 3 * d + 16 + (size_t)(d + 1) * kUPitch;
  const size_t eig = (size_t)(d + 1) * (d + 1) + 3 * d + 16 + 4 * kMaxD + kMaxD + 2 * (kMaxD + 8) + kMaxD;
  return sizeof(double) * (chol > eig ? chol : eig);
}

int ensure_solve_attrs(b2_ctx* ctx) {
  if (!ctx->solve_attr_set) {
    const int bytes = (int)solve_smem_bytes(kMaxD);
    B2_CUDA(cudaFuncSetAttribute(solve_cholesky_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    B2_CUDA(cudaFuncSetAttribute(solve_cholesky_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    B2_CUDA(cudaFuncSetAttribute(solve_spectral_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    B2_CUDA(cudaFuncSetAttribute(solve_eigvals_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    B2_CUDA(cudaFuncSetAttribute(solve_eigh_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)eigh_smem_bytes(kMaxD)));
    B2_CUDA(cudaFuncSetAttribute(solve_enet_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)enet_smem_bytes(kMaxD)));
    B2_CUDA(cudaFuncSetAttribute(bayes_ridge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)bayes_smem_bytes(kMaxD)));
    B2_CUDA(cudaFuncSetAttribute(ard_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ard_smem_bytes(kMaxD)));
    ctx->solve_attr_set = true;
  }
  return B2_OK;
}

}  // namespace

// The Cholesky (LDL^T) kernel writes its result straight into the pinned host mirror (no D2H copy node): the caller
// synchronises the stream and reads ctx->solve_host.
int launch_solve_cholesky(b2_ctx* ctx, double alpha, int fit_intercept, unsigned int gather_epoch) {
  if (int r = ensure_solve_attrs(ctx)) return r;
  SolveXchg xc;
  xc.own = gather_epoch != 0 ? ctx->xchg : nullptr;
  xc.n_ranks = ctx->n_ranks;
  xc.epoch = gather_epoch;
  xc.timeout_ns = ctx->xchg_timeout_ns;
  solve_cholesky_kernel<false><<<1, kCholThreads, solve_smem_bytes(ctx->d), ctx->stream>>>(ctx->S, ctx->d, alpha,
                                                                                           fit_intercept, ctx->solve_host,
                                                                                           xc, nullptr);
  B2_CUDA(cudaGetLastError());
  ctx->launches += 1;
  return B2_OK;
}

int launch_solve_classes(b2_ctx* ctx, double alpha, int fit_intercept, int n_classes) {
  const int T = n_classes == 2 ? 1 : n_classes;
  if (int r = launch_smem(solve_classes_kernel, 1, kClsThreads, (uint32_t)solve_classes_smem_bytes(ctx->d, T),
                          ctx->stream, ctx->S, ctx->d, alpha, fit_intercept, n_classes, ctx->cls))
    return r;
  ctx->launches += 1;
  return B2_OK;
}

int launch_solve_refine(b2_ctx* ctx, double alpha, int fit_intercept) {
  if (int r = ensure_solve_attrs(ctx)) return r;
  SolveXchg xc;
  xc.own = nullptr;
  xc.n_ranks = 1;
  xc.epoch = 0;
  xc.timeout_ns = 0;
  solve_cholesky_kernel<true><<<1, kCholThreads, solve_smem_bytes(ctx->d), ctx->stream>>>(ctx->S, ctx->d, alpha,
                                                                                          fit_intercept, ctx->solve_host,
                                                                                          xc, ctx->refine);
  B2_CUDA(cudaGetLastError());
  ctx->launches += 1;
  return B2_OK;
}

int launch_solve_spectral(b2_ctx* ctx, double cond, int fit_intercept) {
  if (int r = ensure_solve_attrs(ctx)) return r;
  solve_spectral_kernel<<<1, 512, solve_smem_bytes(ctx->d), ctx->stream>>>(ctx->S, ctx->d, cond, fit_intercept, ctx->solve_out);
  B2_CUDA(cudaGetLastError());
  ctx->launches += 1;
  return B2_OK;
}

int launch_solve_eigh(b2_ctx* ctx, int fit_intercept) {
  if (int r = ensure_solve_attrs(ctx)) return r;
  solve_eigh_kernel<<<1, kEighThreads, eigh_smem_bytes(ctx->d), ctx->stream>>>(ctx->S, ctx->d, fit_intercept, ctx->loo);
  B2_CUDA(cudaGetLastError());
  ctx->launches += 1;
  return B2_OK;
}

int launch_solve_enet(b2_ctx* ctx, const EnetArgs& args) {
  if (int r = ensure_solve_attrs(ctx)) return r;
  const int ctas = args.folds != nullptr ? args.n_folds * args.n_l1 : 1;
  solve_enet_kernel<<<ctas, kEnetThreads, enet_smem_bytes(ctx->d), ctx->stream>>>(ctx->S, ctx->d, args);
  B2_CUDA(cudaGetLastError());
  ctx->launches += 1;
  return B2_OK;
}

int launch_bayes_ridge(b2_ctx* ctx, const BayesArgs& args) {
  if (int r = ensure_solve_attrs(ctx)) return r;
  bayes_ridge_kernel<<<1, kByThreads, bayes_smem_bytes(ctx->d), ctx->stream>>>(ctx->S, ctx->d, ctx->loo, args);
  B2_CUDA(cudaGetLastError());
  ctx->launches += 1;
  return B2_OK;
}

int launch_ard(b2_ctx* ctx, const BayesArgs& args) {
  if (int r = ensure_solve_attrs(ctx)) return r;
  ard_kernel<<<1, kByThreads, ard_smem_bytes(ctx->d), ctx->stream>>>(ctx->S, ctx->d, args);
  B2_CUDA(cudaGetLastError());
  ctx->launches += 1;
  return B2_OK;
}

int launch_solve_eigvals(b2_ctx* ctx, double cond, int fit_intercept) {
  if (int r = ensure_solve_attrs(ctx)) return r;
  solve_eigvals_kernel<<<1, kEigThreads, solve_smem_bytes(ctx->d), ctx->stream>>>(ctx->S, ctx->d, cond, fit_intercept,
                                                                                  ctx->solve_out);
  B2_CUDA(cudaGetLastError());
  ctx->launches += 1;
  return B2_OK;
}

}  // namespace b2
