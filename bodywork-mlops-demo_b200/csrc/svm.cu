// svm.cu -- the row pass of the linear SVMs (b2_svm_pass; DESIGN.md section 15).
//
// liblinear's primal trust-region Newton solver (TRON) for the L2-regularised squared hinge (LinearSVC) and squared
// epsilon-insensitive (LinearSVR) losses needs, at each trial point w, the loss, the gradient and the generalized Hessian
// I + 2 C sum z z^T over the rows *active* at w (z = [x 1]).  The pointwise Hessian is 0 or 2 C, so the Hessian at the
// trial point is the one at the accepted point plus sum z z^T over the rows that entered the active set, minus the same
// over the rows that left it.  One pass per call over 32-row tiles, at `from` (the accepted point, or none: the empty set)
// and `to` (the trial point):
//   (1) the tile -> shared memory as z = [x 1 0...] in fp64 from the stored value (exact), zero for rows not kept;
//   (2) eta_from and eta_to per row by the same arithmetic in the same order (the lanes of a warp over the features, a
//       butterfly), so a row's side at `from` is exactly the side the pass that accepted `from` found at its `to`;
//   (3) the pointwise terms at `to` (strict inequalities, as l2r_l2_svc_fun / l2r_l2_svr_fun): squared hinge, t = +-1,
//       m = 1 - t eta, active iff m > 0, loss m^2, g = eta - t; squared epsilon-insensitive, r = eta - y, active iff
//       |r| > eps, e = r -+ eps, loss e^2, g = e; sigma = active_to - active_from;
//   (4) the gradient: thread j adds g_r z_rj over the tile's rows in order (g = 0 where not active);
//   (5) (Hessian) the rows with sigma != 0 are compacted in row order (a ballot and a prefix count) into a staging tile;
//       each time it holds 32 rows, sum sigma z z^T over them on the fp64 tensor core with the upper-block schedule
//       (b2_dmma.cuh: 16 x 16 blocks on and above the diagonal), the partial tile flushed at the end with its unused
//       rows zeroed.  The tensor-core work is proportional to the rows that changed side; sigma z is exact, so the +-
//       sums round only in the additions.
// Each CTA writes its sums in ctx->glm_part in glm_kernel's layout and the ordered reduce adds the CTAs in order: two
// calls return identical sums.
#include "b2_internal.cuh"
#include "b2_dmma.cuh"

namespace b2 {
namespace {

constexpr int kSvBlocks = (kMaxD + 1 + 15) / 16;                                          // 9 blocks of 16 columns
constexpr int kSvSB = (kSvBlocks * (kSvBlocks + 1) / 2 + kTileWarps - 1) / kTileWarps;   // 16 x 16 blocks per warp: 6

__host__ __device__ inline int svm_dp(int d) { return (d + 1 + 15) & ~15; }   // columns of [x 1], padded to 16
size_t svm_smem_bytes(int dp, bool ring, bool hess) {
  const size_t tile = (size_t)kTileRows * tile_vpitch(dp);
  return tile_ring_bytes(ring, true) +
         sizeof(double) * (tile * (hess ? 2 : 1) + 2 * kMaxD + 4 * kTileRows + kTileWarps * 32 + kMaxD + 12) +
         sizeof(int) * (kUpperTable + 2 * kTileRows + 4);
}

// active at eta, and (active) the loss and g: the squared hinge at label sign t, or the squared epsilon-insensitive loss
// of y at p = eps
template <int LOSS>
__device__ __forceinline__ bool svm_active(double eta, double t, double y, double p) {
  if constexpr (LOSS == B2_SVM_SQUARED_HINGE) return 1.0 - t * eta > 0.0;
  else return fabs(eta - y) > p;
}

// Per-CTA sums (glm_kernel's layout): [loss, kept, active at to, entering, leaving, positive, y not finite, 0 | g.z (d + 1),
// zeros | (HESS) the blocks of sum sigma z z^T at kGlmHess, pitch kGlmHp].  op: to = (w, b), from = (step, db),
// misc [2] 1 when from is given, [3] the positive label (squared hinge) or eps (kGlmOp* in b2_internal.cuh).
template <typename T, bool RING, bool HESS, int LOSS>
__global__ void __launch_bounds__(kTileThreads, 1)
svm_kernel(const T* __restrict__ X, int64_t n, int d, int64_t ldx, const float* __restrict__ y,
           const uint8_t* __restrict__ mask, int keep, const double* __restrict__ op, double* __restrict__ part) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  TileRing<T, RING, true> tiles{X, n, d, ldx, y, mask, keep, smem_u32(smem_raw)};
  const int dp = svm_dp(d), zp = tile_vpitch(dp), nb = dp / 16, nsb = nb * (nb + 1) / 2;
  double* Zs = reinterpret_cast<double*>(smem_raw + tile_ring_bytes(RING, true));   // [row][zp]: z = [x 1 0...]
  double* Ss = Zs + (HESS ? kTileRows * zp : 0);   // [slot][zp]: the staged rows that changed side
  double* wv = Ss + kTileRows * zp;        // [kMaxD] w at to
  double* fv = wv + kMaxD;                 // [kMaxD] w at from
  double* yv = fv + kMaxD;                 // y (0 for rows not kept)
  double* gs = yv + kTileRows;             // g (0 for rows not active at to)
  double* sg = gs + kTileRows;             // sigma of the tile's rows
  double* ssg = sg + kTileRows;            // sigma of the staged rows
  double* lsum = ssg + kTileRows;          // [warp][u][8] the scalar sums of the rows warp + 8 u
  double* gsum = lsum + kTileWarps * 32;   // [kMaxD + 8] the gradient sums, entry j of thread j
  double* msc = gsum + kMaxD + 8;          // [4] b at to, b at from, 1 when from is given, the label or eps
  int* sb = reinterpret_cast<int*>(msc + 4);   // the upper blocks' table
  int* dst = sb + kUpperTable;             // the staging slot of each changed row (-1: unchanged), past 31: next round
  int* kp = dst + kTileRows;               // 1 for the tile's kept rows
  int* cnt = kp + kTileRows;              // [0] rows in the staging tile, [1] the same plus the tile's changed rows
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g8 = lane >> 2, t4 = lane & 3;
  for (int t = tid; t < kTileWarps * 32; t += blockDim.x) lsum[t] = 0.0;
  for (int t = tid; t < kMaxD + 8; t += blockDim.x) gsum[t] = 0.0;
  if (tid < 4) msc[tid] = op[kGlmOpMisc + tid];   // read where used: the registers go to the Hessian's accumulators
  for (int t = tid; t < kMaxD; t += blockDim.x) {
    wv[t] = t < d ? op[kGlmOpW + t] : 0.0;
    fv[t] = t < d ? op[kGlmOpStep + t] : 0.0;
  }
  if (tid == 0) cnt[0] = 0;
  upper_blocks(sb, nb);
  const int64_t n_tiles = (n + kTileRows - 1) / kTileRows;
  tiles.start();
  double acc[kSvSB][4][2] = {};                     // (HESS) the warp's blocks, held for the whole launch
  // H += (sigma z)^T z over the 32 staged rows, the warp's blocks
  auto flush = [&]() {
    upper_accumulate(acc, sb, nsb, [&](int r, int c) { return ssg[r] * Ss[r * zp + c]; }, Ss, zp, warp, g8, t4);
  };
  if (!tiles.produce()) {
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
      // (1) the tile: z = [x 1 0...] and y, zero for rows not kept
      tiles.load(tile * kTileRows, dp,
                 [&](int r, int j, bool kept, bool live, float x) {
                   Zs[r * zp + j] = live ? (double)x : (kept && j == d ? 1.0 : 0.0);
                 },
                 [&](int r, bool kept, double yr) {
                   yv[r] = yr;
                   kp[r] = kept;
                 });
      __syncwarp();
      // (2) eta at to and at from of the warp's rows, the same arithmetic; lane u keeps row warp + 8 u's
      double e = 0.0, ef = 0.0;
#pragma unroll
      for (int u = 0; u < kTileRowsPerWarp; ++u) {
        const double* zr = Zs + (warp + kTileWarps * u) * zp;
        double a = 0.0, c = 0.0;
        for (int j = lane; j < d; j += 32) {
          a = fma(zr[j], wv[j], a);
          c = fma(zr[j], fv[j], c);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          a += __shfl_xor_sync(0xffffffffu, a, o);
          c += __shfl_xor_sync(0xffffffffu, c, o);
        }
        if (lane == u) {
          e = a + msc[0];
          ef = c + msc[1];
        }
      }
      // (3) the pointwise terms: lane u takes row warp + 8 u
      if (lane < kTileRowsPerWarp) {
        const int r = warp + kTileWarps * lane;
        const bool kept = kp[r] != 0;
        const double yy = yv[r], param = msc[3];
        const bool pos = yy == param;
        const double t = pos ? 1.0 : -1.0;
        const bool act = kept && svm_active<LOSS>(e, t, yy, param);
        const bool act_f = kept && msc[2] != 0.0 && svm_active<LOSS>(ef, t, yy, param);
        double l, gg;
        if constexpr (LOSS == B2_SVM_SQUARED_HINGE) {
          const double m = 1.0 - t * e;
          l = m * m;
          gg = e - t;
        } else {
          const double rr = e - yy;
          gg = rr > param ? rr - param : rr + param;
          l = gg * gg;
        }
        double* ls = lsum + (warp * 4 + lane) * 8;
        ls[0] += act ? l : 0.0;
        ls[1] += kept ? 1.0 : 0.0;
        ls[2] += act ? 1.0 : 0.0;
        ls[3] += (act && !act_f) ? 1.0 : 0.0;
        ls[4] += (act_f && !act) ? 1.0 : 0.0;
        ls[5] += (LOSS == B2_SVM_SQUARED_HINGE && kept && pos) ? 1.0 : 0.0;
        ls[6] += (kept && !isfinite(yy)) ? 1.0 : 0.0;
        gs[r] = act ? gg : 0.0;
        sg[r] = (double)((int)act - (int)act_f);
      }
      tile_consumer_sync();
      // (4) the gradient
      if (tid <= d) {
        double a = gsum[tid];
#pragma unroll 8
        for (int r = 0; r < kTileRows; ++r) a = fma(gs[r], Zs[r * zp + tid], a);
        gsum[tid] = a;
      }
      if constexpr (HESS) {
        // (5) the changed rows in row order: slot staged + their rank among the tile's changed rows
        if (warp == 0) {
          const int staged = cnt[0];
          const bool chg = sg[lane] != 0.0;
          const unsigned bal = __ballot_sync(0xffffffffu, chg);
          dst[lane] = chg ? staged + __popc(bal & ((1u << lane) - 1u)) : -1;
          if (lane == 0) {                          // the staged rows after this tile: total, or total - 32 past a flush
            cnt[1] = staged + __popc(bal);
            cnt[0] = cnt[1] & (kTileRows - 1);
          }
        }
        tile_consumer_sync();
        const int total = cnt[1];
        for (int t = tid; t < kTileRows * dp; t += kTileConsumers) {
          const int r = t / dp, j = t - r * dp, p = dst[r];
          if (p >= 0 && p < kTileRows) {
            Ss[p * zp + j] = Zs[r * zp + j];
            if (j == 0) ssg[p] = sg[r];
          }
        }
        if (total >= kTileRows) {
          tile_consumer_sync();
          flush();
          tile_consumer_sync();
          for (int t = tid; t < kTileRows * dp; t += kTileConsumers) {
            const int r = t / dp, j = t - r * dp, p = dst[r] - kTileRows;
            if (p >= 0) {
              Ss[p * zp + j] = Zs[r * zp + j];
              if (j == 0) ssg[p] = sg[r];
            }
          }
        }
      }
      tile_consumer_sync();
    }
    if constexpr (HESS) {
      const int staged = cnt[0];
      if (staged > 0) {                             // the partial staging tile, its unused rows zeroed
        for (int t = tid; t < (kTileRows - staged) * zp; t += kTileConsumers) Ss[staged * zp + t] = 0.0;
        for (int t = staged + tid; t < kTileRows; t += kTileConsumers) ssg[t] = 0.0;
        tile_consumer_sync();
        flush();
      }
    }
  }
  // the CTA's sums in a fixed order: the lanes of a warp, then the warps in order
  double* out = part + (size_t)blockIdx.x * kGlmPart;
  __syncthreads();
  if (tid < kGlmHess) {                             // the scalars, the gradient, zeros in the unused entries
    double r = 0.0;
    if (tid < 7)
      for (int q = 0; q < kTileWarps * 4; ++q) r += lsum[q * 8 + tid];
    else if (tid >= kGlmGrad && tid <= kGlmGrad + d)
      r = gsum[tid - kGlmGrad];
    out[tid] = r;
  }
  if constexpr (HESS) upper_store(acc, sb, nsb, out + kGlmHess, kGlmHp, warp, g8, t4);
}

}  // namespace

// The rows [0, n) in split_ring_rows's launches, each followed by the ordered reduce into ctx->glm (`first_block`
// overwrites, otherwise adds).  Without the Hessian two CTAs per SM hide the latency of the per-tile steps.
int launch_svm(b2_ctx* ctx, const void* X, int x_dtype, int64_t n, int d, int64_t ldx, const float* y,
               const uint8_t* mask, int keep, int loss, bool hess, bool first_block) {
  return split_ring_rows(ctx, X, x_dtype, n, d, ldx, y, mask, kTileRows, first_block, [&](bool ring, const RowSpan& s) {
    const int grid = tile_grid(s.rows, ctx->sm_count, hess ? 1 : 2);
    const uint32_t smem = (uint32_t)svm_smem_bytes(svm_dp(d), ring, hess);
    const int rc = with_rows(x_dtype, s.X, [&](auto* Xr) {
      using T = row_t<decltype(Xr)>;
      return with_int<0, 1>((int)hess, [&](auto H) {
        return with_int<B2_SVM_SQUARED_HINGE, B2_SVM_SQUARED_EPSILON>(loss, [&](auto L) {
          constexpr bool HESS = decltype(H)::value == 1;
          constexpr int LOSS = decltype(L)::value;
          auto kernel = ring ? svm_kernel<T, true, HESS, LOSS> : svm_kernel<T, false, HESS, LOSS>;
          return launch_smem(kernel, grid, tile_threads(ring), smem, ctx->stream, Xr, s.rows, d, ldx, s.y, s.mask,
                             keep, static_cast<const double*>(ctx->glm + kGlmOp), ctx->glm_part);
        });
      });
    });
    if (rc != B2_OK) return rc;
    return launch_ordered_reduce(ctx, ctx->glm_part, kGlmPart, grid, s.first, kGlmHess, 0u, ctx->glm,
                                 hess ? d + 1 : 0, kGlmHess, kGlmHp);
  });
}

}  // namespace b2
