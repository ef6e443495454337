// score_std.cu -- the predictive standard deviation of BayesianRidge / ARDRegression (b2_score_std; DESIGN.md section 9).
//
// Per row, with v = x - m: ystd = sqrt(max(v^T sigma v, 0) + noise_var) and yhat = v.w + (b + m.w), scikit-learn's
// predict(X, return_std=True).  That is 2 D^2 flops against D * 4 bytes of row: the pass is fp64-compute bound, so the
// product runs on the fp64 tensor core (mma.sync m8n8k4 f64), as the leave-one-out pass (ridge_loo.cu) does:
//   (1) a tile of 32 rows -> shared memory as v = x - m in fp64 from the stored value (one rounding);
//   (2) Z = V [sigma | w], the B operand resident in shared memory for the whole launch (column dp holds w);
//   (3) each lane multiplies its accumulators by the matching v and the four lanes of a row add theirs, then the warps are
//       added in warp order: q = rowsum(Z o V).  The lane that holds column dp writes V w.
// The rows take scoring's plan (plan_rows): contiguous 16-byte aligned rows arrive in whole 32-row tiles through the
// bulk-copy ring (ring_produce), the rows after the last whole tile and every other layout are read by the same consumers
// from global memory.  Every sum runs in a fixed order, so repeated calls give identical results.
#include "b2_internal.cuh"
#include "b2_dmma.cuh"

namespace b2 {
namespace {

constexpr int kStdNT = 3;   // n-tiles per warp: (128 + 8) / 8 = 17 <= 3 * 8

// the B operand [sigma | w] has dp + 8 columns: sigma, then w and zeros
size_t std_smem_bytes(int dp, bool ring) {
  return tile_ring_bytes(ring, false) +
         sizeof(double) * ((size_t)dp * tile_bpitch(dp) + (size_t)kTileRows * tile_vpitch(dp) + kTileWarps * kTileRows +
                           kTileRows + kMaxD);
}

// RING: rows [0, n), n a multiple of kTileRows, contiguous (ldx == d) and 16-byte aligned, through the bulk-copy ring;
// otherwise rows [0, n) of any layout from global memory.  Tiles blockIdx.x, + gridDim.x, ...  op: ctx->enet (kStd*).
template <typename T, bool RING>
__global__ void __launch_bounds__(kTileThreads, 1)
score_std_kernel(const T* __restrict__ X, int64_t n, int d, int64_t ldx, const double* __restrict__ op,
                 double* __restrict__ yhat, double* __restrict__ ystd) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  TileRing<T, RING, false> tiles{X, n, d, ldx, nullptr, nullptr, 0, smem_u32(smem_raw)};
  const int dp = tile_dp(d), bp = tile_bpitch(dp), vp = tile_vpitch(dp), ntc = dp / 8 + 1;
  double* Bs = reinterpret_cast<double*>(smem_raw + tile_ring_bytes(RING, false));   // [dp][bp]: sigma | w, zero padded
  double* Vs = Bs + dp * bp;               // the tile: v = x - m
  double* qpart = Vs + kTileRows * vp;     // [warp][row] partial quadratic forms
  double* yv = qpart + kTileWarps * kTileRows;   // V w per row
  double* mean = yv + kTileRows;           // [kMaxD]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t4 = lane & 3;
  for (int t = tid; t < dp * bp; t += blockDim.x) {
    const int i = t / bp, k = t - i * bp;
    double v = 0.0;
    if (i < d && k < d) v = op[kStdSigma + i * d + k];
    else if (i < d && k == dp) v = op[kStdCoef + i];
    Bs[t] = v;
  }
  for (int t = tid; t < kMaxD; t += blockDim.x) mean[t] = t < d ? op[kStdMean + t] : 0.0;
  const double b_eff = op[kStdMisc], noise_var = op[kStdMisc + 1];
  const int64_t n_tiles = (n + kTileRows - 1) / kTileRows;
  tiles.start();
  if (tiles.produce()) return;
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int64_t row0 = tile * kTileRows;
    // (1) the tile: v = x - m
    tiles.load(row0, dp,
               [&](int r, int j, bool, bool live, float x) { Vs[r * vp + j] = live ? (double)x - mean[j] : 0.0; },
               [](int, bool, double) {});
    tile_consumer_sync();
    // (2) Z = V B: warp w takes the n-tiles w, w + 8, w + 16 of the dp / 8 + 1, all m-tiles
    double z[kStdNT][kTileMT][2];
    tile_product(Vs, vp, Bs, bp, dp, ntc, z);
    // (3) the lane's share of q per row, then the four lanes of the row
    double qp[kTileMT];
#pragma unroll
    for (int mt = 0; mt < kTileMT; ++mt) qp[mt] = 0.0;
#pragma unroll
    for (int u = 0; u < kStdNT; ++u) {
      const int nt = warp + kTileWarps * u;
      if (nt < dp / 8) {
        const int c0 = 8 * nt + 2 * t4;
#pragma unroll
        for (int mt = 0; mt < kTileMT; ++mt) {
          const double* vr = Vs + (8 * mt + g) * vp + c0;
          qp[mt] = fma(z[u][mt][0], vr[0], qp[mt]);
          qp[mt] = fma(z[u][mt][1], vr[1], qp[mt]);
        }
      } else if (nt == dp / 8 && t4 == 0) {
#pragma unroll
        for (int mt = 0; mt < kTileMT; ++mt) yv[8 * mt + g] = z[u][mt][0];
      }
    }
#pragma unroll
    for (int mt = 0; mt < kTileMT; ++mt) {
      double v = qp[mt];
      v += __shfl_xor_sync(0xffffffffu, v, 1);
      v += __shfl_xor_sync(0xffffffffu, v, 2);
      if (t4 == 0) qpart[warp * kTileRows + 8 * mt + g] = v;
    }
    tile_consumer_sync();
    if (tid < kTileRows) {
      const int64_t row = row0 + tid;
      if (row < n) {
        double q = 0.0;
        for (int w = 0; w < kTileWarps; ++w) q += qpart[w * kTileRows + tid];
        ystd[row] = sqrt(fmax(q, 0.0) + noise_var);
        if (yhat != nullptr) yhat[row] = yv[tid] + b_eff;
      }
    }
    tile_consumer_sync();
  }
}

}  // namespace

// The rows [0, n) in the launches of scoring's plan: the whole 32-row tiles of what plan_rows streams through the ring go
// to the ring flavour, the rest (or every row of another layout) to the direct one.
int launch_score_std(b2_ctx* ctx, const void* X, int x_dtype, int64_t n, int d, int64_t ldx, double* yhat, double* ystd) {
  // no sums: `first` is false, so a part without rows is never launched
  const auto part = [&](bool ring, const RowSpan& s) {
    const int grid = tile_grid(s.rows, ctx->sm_count, 1);
    double* yh = yhat != nullptr ? yhat + s.r0 : nullptr;
    const uint32_t smem = (uint32_t)std_smem_bytes(tile_dp(d), ring);
    const int rc = with_rows(x_dtype, s.X, [&](auto* Xr) {
      using T = row_t<decltype(Xr)>;
      auto kernel = ring ? score_std_kernel<T, true> : score_std_kernel<T, false>;
      return launch_smem(kernel, grid, tile_threads(ring), smem, ctx->stream, Xr, s.rows, d, ldx,
                         static_cast<const double*>(ctx->enet), yh, ystd + s.r0);
    });
    if (rc != B2_OK) return rc;
    ctx->launches += 1;
    return B2_OK;
  };
  return split_ring_rows(ctx, X, x_dtype, n, d, ldx, nullptr, nullptr, kTileRows, false, part);
}

}  // namespace b2
