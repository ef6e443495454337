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
#include "b2_ptx.cuh"

namespace b2 {
namespace {

constexpr int kStdRows = 32;                        // rows per tile
constexpr int kStdMT = kStdRows / 8;                // m-tiles of the DMMA per tile
constexpr int kStdWarps = 8;                        // consumer warps
constexpr int kStdConsumers = 32 * kStdWarps;
constexpr int kStdThreads = kStdConsumers + 32;     // + the producer warp of the ring
constexpr int kStdStages = 3;
constexpr int kStdNT = 3;                           // n-tiles per warp: (128 + 8) / 8 = 17 <= 3 * 8
constexpr uint32_t kStdXStage = kStdRows * kMaxD * 4;                      // 16 KB: 32 fp32 rows of 128 features
constexpr uint32_t kStdOffBar = kStdStages * kStdXStage;
constexpr uint32_t kStdRingBytes = kStdOffBar + 2 * kStdStages * 8 + 16;    // the doubles start here (16-byte aligned)

__host__ __device__ inline int std_dp(int d) { return (d + 7) & ~7; }
__host__ __device__ inline int std_bpitch(int dp) { return dp + 8; }       // dp + 8 columns: sigma, then w and zeros
__host__ __device__ inline int std_vpitch(int dp) { return dp + 4; }
size_t std_smem_bytes(int dp, bool ring) {
  return (ring ? kStdRingBytes : 0) +
         sizeof(double) * ((size_t)dp * std_bpitch(dp) + (size_t)kStdRows * std_vpitch(dp) + kStdWarps * kStdRows +
                           kStdRows + kMaxD);
}

__device__ __forceinline__ void consumer_sync() {   // the consumer warps only (the producer is inside ring_produce)
  asm volatile("bar.sync 1, %0;" ::"r"(kStdConsumers) : "memory");
}

// RING: rows [0, n), n a multiple of kStdRows, contiguous (ldx == d) and 16-byte aligned, through the bulk-copy ring;
// otherwise rows [0, n) of any layout from global memory.  Tiles blockIdx.x, + gridDim.x, ...  op: ctx->enet (kStd*).
template <typename T, bool RING>
__global__ void __launch_bounds__(kStdThreads, 1)
score_std_kernel(const T* __restrict__ X, int64_t n, int d, int64_t ldx, const double* __restrict__ op,
                 double* __restrict__ yhat, double* __restrict__ ystd) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const uint32_t sbase = smem_u32(smem_raw);
  const uint32_t bar_full = sbase + kStdOffBar, bar_empty = bar_full + 8 * kStdStages;
  const int dp = std_dp(d), bp = std_bpitch(dp), vp = std_vpitch(dp), ntc = dp / 8 + 1;
  double* Bs = reinterpret_cast<double*>(smem_raw + (RING ? kStdRingBytes : 0));   // [dp][bp]: sigma | w, zero padded
  double* Vs = Bs + dp * bp;               // the tile: v = x - m
  double* qpart = Vs + kStdRows * vp;      // [warp][row] partial quadratic forms
  double* yv = qpart + kStdWarps * kStdRows;   // V w per row
  double* mean = yv + kStdRows;            // [kMaxD]
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
  const int64_t n_tiles = (n + kStdRows - 1) / kStdRows;
  if constexpr (RING) ring_init<kStdStages>(bar_full, bar_empty, kStdWarps);   // includes a block barrier
  else __syncthreads();
  if (RING && warp == kStdWarps) {
    if (lane == 0)
      ring_produce<kStdStages>(bar_full, bar_empty, (int)n_tiles, kStdRows, X, (uint32_t)(d * sizeof(T)), sbase,
                               kStdXStage, false, nullptr, 0u, 0u, false, nullptr, 0u, 0u);
    return;
  }
  int s = 0;
  uint32_t phase = 0;
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int64_t row0 = tile * kStdRows;
    // (1) the tile
    if constexpr (RING) {
      mbar_wait(bar_full + 8 * s, phase);
      const uint32_t xs = sbase + s * kStdXStage;
#pragma unroll
      for (int u = 0; u < kStdRows / kStdWarps; ++u) {
        const int r = warp + kStdWarps * u;
        const uint32_t xr = xs + (uint32_t)(r * d) * (uint32_t)sizeof(T);
        for (int j = lane; j < dp; j += 32) {
          const bool live = j < d;
          const float x = live ? raw_ld_shared<T>(xr + (uint32_t)j * (uint32_t)sizeof(T)) : 0.f;
          Vs[r * vp + j] = live ? (double)x - mean[j] : 0.0;
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_empty + 8 * s);      // the slot is converted: the producer may refill it
      if (++s == kStdStages) { s = 0; phase ^= 1u; }
    } else {
      for (int r = warp; r < kStdRows; r += kStdWarps) {
        const int64_t row = row0 + r;
        const bool use = row < n;
        const T* xr = X + row * ldx;
        for (int j = lane; j < dp; j += 32) {
          const bool live = use && j < d;
          const float x = live ? ld_row_val<T>(xr + j) : 0.f;
          Vs[r * vp + j] = live ? (double)x - mean[j] : 0.0;
        }
      }
    }
    consumer_sync();
    // (2) Z = V B: warp w takes the n-tiles w, w + 8, w + 16 of the dp / 8 + 1, all m-tiles
    double z[kStdNT][kStdMT][2];
#pragma unroll
    for (int u = 0; u < kStdNT; ++u) {
#pragma unroll
      for (int mt = 0; mt < kStdMT; ++mt) { z[u][mt][0] = 0.0; z[u][mt][1] = 0.0; }
      const int nt = warp + kStdWarps * u;
      if (nt < ntc) {
        for (int ks = 0; ks < dp / 4; ++ks) {
          const double b = Bs[(4 * ks + t4) * bp + 8 * nt + g];
          double a[kStdMT];
#pragma unroll
          for (int mt = 0; mt < kStdMT; ++mt) a[mt] = Vs[(8 * mt + g) * vp + 4 * ks + t4];
#pragma unroll
          for (int mt = 0; mt < kStdMT; ++mt) dmma(z[u][mt][0], z[u][mt][1], a[mt], b);
        }
      }
    }
    // (3) the lane's share of q per row, then the four lanes of the row
    double qp[kStdMT];
#pragma unroll
    for (int mt = 0; mt < kStdMT; ++mt) qp[mt] = 0.0;
#pragma unroll
    for (int u = 0; u < kStdNT; ++u) {
      const int nt = warp + kStdWarps * u;
      if (nt < dp / 8) {
        const int c0 = 8 * nt + 2 * t4;
#pragma unroll
        for (int mt = 0; mt < kStdMT; ++mt) {
          const double* vr = Vs + (8 * mt + g) * vp + c0;
          qp[mt] = fma(z[u][mt][0], vr[0], qp[mt]);
          qp[mt] = fma(z[u][mt][1], vr[1], qp[mt]);
        }
      } else if (nt == dp / 8 && t4 == 0) {
#pragma unroll
        for (int mt = 0; mt < kStdMT; ++mt) yv[8 * mt + g] = z[u][mt][0];
      }
    }
#pragma unroll
    for (int mt = 0; mt < kStdMT; ++mt) {
      double v = qp[mt];
      v += __shfl_xor_sync(0xffffffffu, v, 1);
      v += __shfl_xor_sync(0xffffffffu, v, 2);
      if (t4 == 0) qpart[warp * kStdRows + 8 * mt + g] = v;
    }
    consumer_sync();
    if (tid < kStdRows) {
      const int64_t row = row0 + tid;
      if (row < n) {
        double q = 0.0;
        for (int w = 0; w < kStdWarps; ++w) q += qpart[w * kStdRows + tid];
        ystd[row] = sqrt(fmax(q, 0.0) + noise_var);
        if (yhat != nullptr) yhat[row] = yv[tid] + b_eff;
      }
    }
    consumer_sync();
  }
}

}  // namespace

// The rows [0, n) in the launches of scoring's plan: the whole 32-row tiles of what plan_rows streams through the ring go
// to the ring flavour, the rest (or every row of another layout) to the direct one.
int launch_score_std(b2_ctx* ctx, const void* X, int x_dtype, int64_t n, int d, int64_t ldx, double* yhat, double* ystd) {
  // no sums: `first` is false, so a part without rows is never launched
  return split_ring_rows(ctx, X, x_dtype, n, d, ldx, nullptr, nullptr, kStdRows, false, [&](bool ring, const RowSpan& s) {
    const int64_t n_tiles = (s.rows + kStdRows - 1) / kStdRows;
    const int grid = (int)(n_tiles < ctx->sm_count ? n_tiles : ctx->sm_count);
    double* yh = yhat != nullptr ? yhat + s.r0 : nullptr;
    const uint32_t smem = (uint32_t)std_smem_bytes(std_dp(d), ring);
    const int rc = with_rows(x_dtype, s.X, [&](auto* Xr) {
      using T = row_t<decltype(Xr)>;
      auto kernel = ring ? score_std_kernel<T, true> : score_std_kernel<T, false>;
      return launch_smem(kernel, grid, ring ? kStdThreads : kStdConsumers, smem, ctx->stream, Xr, s.rows, d, ldx,
                         static_cast<const double*>(ctx->enet), yh, ystd + s.r0);
    });
    if (rc != B2_OK) return rc;
    ctx->launches += 1;
    return B2_OK;
  });
}

}  // namespace b2
