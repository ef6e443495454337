// solve.cu -- single-SM fp64 solve of the centred (ridge) normal equations from S.
//
// Replaces scipy.linalg.lstsq + _set_intercept inside LinearRegression.fit
// (stage_1_train_model.py:105-106 -> sklearn/linear_model/_base.py: `linalg.lstsq(Xc, yc, cond=tol)`
// then `intercept_ = y_offset - X_offset @ coef_`).  Ridge term as sklearn/linear_model/_ridge.py
// (`(Xc^T Xc + alpha I) w = Xc^T yc`).
//
//   solve_cholesky_kernel : A = Xc^T Xc + alpha I = L L^T in shared memory, two triangular solves.
//   solve_spectral_kernel : one-sided Jacobi on A (A V = W, columns of W orthogonal => w_k = lambda_k v_k):
//                           singular_ = sqrt(lambda) (descending), rank_ = #{sqrt(lambda) > cond * max},
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

// Builds A (pitch d+1) and r in shared memory from the raw statistic; returns means.  S is read through L2 (__ldcg: the
// fused solve has just written it from this CTA) with the loads of a whole batch issued before the first use -- the
// phase is two L2 round trips, not one per element.
__device__ void build_normal_equations(const double* S, int d, double alpha, int fit_intercept,
                                       double* A, double* r, double* mean, double* ybar_out) {
  const int dp = d + 2, pitch = d + 1;
  const double n = __ldcg(S + d * dp + d);
  const double inv_n = n > 0.0 ? 1.0 / n : 0.0;
  double sxy = 0.0;
  if ((int)threadIdx.x < d) {
    const double sx = __ldcg(S + threadIdx.x * dp + d);
    sxy = __ldcg(S + threadIdx.x * dp + d + 1);
    mean[threadIdx.x] = fit_intercept ? sx * inv_n : 0.0;
  }
  const double ybar = fit_intercept ? __ldcg(S + d * dp + d + 1) * inv_n : 0.0;
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
      v[u] = j < d ? __ldcg(S + i0 * dp + j) : 0.0;
      v[4 + u] = (j < d && i1 < d) ? __ldcg(S + i1 * dp + j) : 0.0;
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

__global__ void __launch_bounds__(kCholThreads, 1)
solve_cholesky_kernel(double* S, int d, double alpha, int fit_intercept, double* __restrict__ out, const SolveXchg xc) {
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
  // eigenvalues = column norms
  for (int k = threadIdx.x; k < d; k += blockDim.x) {
    double s2 = 0.0;
    for (int row = 0; row < d; ++row) s2 += W[k * pitch + row] * W[k * pitch + row];
    lam[k] = sqrt(s2);
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

size_t solve_smem_bytes(int d) {
  // Cholesky: A, mean, invd, misc, U panel; eigenvalue kernel: A, r, mean, misc, (v, w) x 2, pv, dd, ee2, lam
  const size_t chol = (size_t)(d + 1) * (d + 1) + 3 * d + 16 + (size_t)(d + 1) * kUPitch;
  const size_t eig = (size_t)(d + 1) * (d + 1) + 3 * d + 16 + 4 * kMaxD + kMaxD + 2 * (kMaxD + 8) + kMaxD;
  return sizeof(double) * (chol > eig ? chol : eig);
}

int ensure_solve_attrs(b2_ctx* ctx) {
  if (!ctx->solve_attr_set) {
    const int bytes = (int)solve_smem_bytes(kMaxD);
    B2_CUDA(cudaFuncSetAttribute(solve_cholesky_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    B2_CUDA(cudaFuncSetAttribute(solve_spectral_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    B2_CUDA(cudaFuncSetAttribute(solve_eigvals_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
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
  solve_cholesky_kernel<<<1, kCholThreads, solve_smem_bytes(ctx->d), ctx->stream>>>(ctx->S, ctx->d, alpha, fit_intercept,
                                                                                    ctx->solve_host, xc);
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

int launch_solve_eigvals(b2_ctx* ctx, double cond, int fit_intercept) {
  if (int r = ensure_solve_attrs(ctx)) return r;
  solve_eigvals_kernel<<<1, kEigThreads, solve_smem_bytes(ctx->d), ctx->stream>>>(ctx->S, ctx->d, cond, fit_intercept,
                                                                                  ctx->solve_out);
  B2_CUDA(cudaGetLastError());
  ctx->launches += 1;
  return B2_OK;
}

}  // namespace b2
