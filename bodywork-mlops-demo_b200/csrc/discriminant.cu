// discriminant.cu -- the within-class scatter pass of LinearDiscriminantAnalysis (b2_class_scatter; DESIGN.md section 16).
//
// Every solver of scikit-learn's LinearDiscriminantAnalysis needs, beyond the class counts and means (b2_class_sums),
// the pooled within-class scatter weighted per class, S_w(w) = sum over the kept rows of w_y (x - m_y)(x - m_y)^T (the
// priors' covariance is S_w(p_k / n_k), the svd solver's and the total scatter's S_w(1)).  Building it from the Gram
// minus the class means would cancel the squared column offsets against the within-class variance, so one fp64 pass
// centres each row on its class mean first.  One pass per call over 32-row tiles:
//   (1) the tile -> shared memory as x in fp64 from the stored value (exact), and each row's class (its index in the
//       sorted classes, -1 for a kept row of no class, NaN included, -2 for a row not kept); lane 0 of each warp counts
//       its rows;
//   (2) u = x - m_class in fp64, zero for rows of no class and rows not kept, and A = w_class u beside it;
//   (3) S_w += A^T u on the fp64 tensor core with the upper-block schedule (b2_dmma.cuh): 16 x 16 blocks on and above
//       the diagonal (36 at D = 128: there is no intercept column), each warp holding up to five of them for the whole
//       launch, the 8 x 8 tile below the diagonal of a diagonal block skipped.
// The class means (at most 32 x 128 doubles) sit in shared memory beside the tile for the whole launch.  Each CTA writes
// its sums in ctx->disc_part and the ordered reduce adds the CTAs in order: two calls return identical sums.
#include "b2_internal.cuh"
#include "b2_dmma.cuh"

namespace b2 {
namespace {

constexpr int kDaBlocks = kMaxD / 16;                                                      // 8 blocks of 16 columns
constexpr int kDaSB = (kDaBlocks * (kDaBlocks + 1) / 2 + kTileWarps - 1) / kTileWarps;   // 16 x 16 blocks per warp: 5

__host__ __device__ inline int scatter_dp(int d) { return (d + 15) & ~15; }   // the features, padded to 16
// the ring, the tile u and w u [2][kTileRows][zp], the means [K][dp], the weights, the warps' counts [kTileWarps][4],
// the classes, the rows' classes and the blocks on and above the diagonal
size_t scatter_smem_bytes(int dp, int n_classes, bool ring) {
  return tile_ring_bytes(ring, true) +
         sizeof(double) * (2 * (size_t)kTileRows * tile_vpitch(dp) + (size_t)n_classes * dp + kMaxClasses +
                           kTileWarps * 4) +
         sizeof(float) * kMaxClasses + sizeof(int) * (kTileRows + kUpperTable);
}

// Per CTA: [0] kept rows [1] kept rows of no class [2] kept rows with y not finite, zeros to kDaHead, then the upper
// blocks of sum w u u^T at kDaHead + i kMaxD + j.  op: ctx->disc.
template <typename T, bool RING>
__global__ void __launch_bounds__(kTileThreads, 1)
class_scatter_kernel(const T* __restrict__ X, int64_t n, int d, int64_t ldx, const float* __restrict__ y,
                     const uint8_t* __restrict__ mask, int keep, int n_classes, const double* __restrict__ op,
                     double* __restrict__ part) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  TileRing<T, RING, true> tiles{X, n, d, ldx, y, mask, keep, smem_u32(smem_raw)};
  const int dp = scatter_dp(d), zp = tile_vpitch(dp), nb = dp / 16, nsb = nb * (nb + 1) / 2, K = n_classes;
  double* Us = reinterpret_cast<double*>(smem_raw + tile_ring_bytes(RING, true));   // [row][zp]: x, then u
  double* As = Us + kTileRows * zp;        // [row][zp]: w u
  double* Ms = As + kTileRows * zp;        // [K][dp]: the class means, zero padded
  double* wv = Ms + K * dp;                // [kMaxClasses] the class weights
  double* cnt = wv + kMaxClasses;          // [warp][4]: kept, no class, y not finite
  float* cls = reinterpret_cast<float*>(cnt + kTileWarps * 4);
  int* row_class = reinterpret_cast<int*>(cls + kMaxClasses);
  int* sb = row_class + kTileRows;         // the upper blocks' table
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g8 = lane >> 2, t4 = lane & 3;
  for (int t = tid; t < K * dp; t += blockDim.x) {
    const int k = t / dp, j = t - k * dp;
    Ms[t] = j < d ? op[kDaMeans + k * kMaxD + j] : 0.0;
  }
  for (int t = tid; t < kMaxClasses; t += blockDim.x) {
    wv[t] = t < K ? op[kDaWeights + t] : 0.0;
    cls[t] = t < K ? (float)op[kDaClasses + t] : 0.f;
  }
  for (int t = tid; t < kTileWarps * 4; t += blockDim.x) cnt[t] = 0.0;
  upper_blocks(sb, nb);
  const int64_t n_tiles = (n + kTileRows - 1) / kTileRows;
  tiles.start();
  double acc[kDaSB][4][2] = {};            // the warp's blocks, held for the whole launch
  if (!tiles.produce()) {
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
      // (1) the tile and the rows' classes
      tiles.load(tile * kTileRows, dp,
                 [&](int r, int j, bool, bool live, float x) { Us[r * zp + j] = live ? (double)x : 0.0; },
                 [&](int r, bool kept, double yr) {
                   const int k = kept ? class_of(cls, K, (float)yr) : -2;
                   row_class[r] = k;
                   double* c = cnt + warp * 4;
                   c[0] += kept ? 1.0 : 0.0;
                   c[1] += k == -1 ? 1.0 : 0.0;
                   c[2] += (kept && !isfinite(yr)) ? 1.0 : 0.0;
                 });
      tile_consumer_sync();
      // (2) u = x - m_class and w u, zero for the rows of no class
      for (int t = tid; t < kTileRows * dp; t += kTileConsumers) {
        const int r = t / dp, j = t - r * dp, k = row_class[r];
        const double u = k >= 0 ? Us[r * zp + j] - Ms[k * dp + j] : 0.0;
        Us[r * zp + j] = u;
        As[r * zp + j] = k >= 0 ? wv[k] * u : 0.0;
      }
      tile_consumer_sync();
      // (3) S_w += (w u)^T u over the tile's rows, the warp's blocks
      upper_accumulate(acc, sb, nsb, [&](int r, int c) { return As[r * zp + c]; }, Us, zp, warp, g8, t4);
      tile_consumer_sync();
    }
  }
  // the CTA's sums in a fixed order: the warps' counts in warp order, the blocks as the warps hold them
  double* out = part + (size_t)blockIdx.x * kDaPart;
  __syncthreads();
  if (tid < kDaHead) {
    double v = 0.0;
    if (tid < 3)
      for (int w = 0; w < kTileWarps; ++w) v += cnt[w * 4 + tid];
    out[tid] = v;
  }
  upper_store(acc, sb, nsb, out + kDaHead, kMaxD, warp, g8, t4);
}

}  // namespace

// The rows [0, n) in split_ring_rows's launches, each followed by the ordered reduce into ctx->disc + kDaSums
// (`first_block` overwrites, otherwise adds).  One CTA per SM: the accumulators take the registers of two.
int launch_class_scatter(b2_ctx* ctx, const void* X, int x_dtype, int64_t n, int d, int64_t ldx, const float* y,
                         const uint8_t* mask, int keep, int n_classes, bool first_block) {
  return split_ring_rows(ctx, X, x_dtype, n, d, ldx, y, mask, kTileRows, first_block, [&](bool ring, const RowSpan& s) {
    const int grid = tile_grid(s.rows, ctx->sm_count, 1);
    const uint32_t smem = (uint32_t)scatter_smem_bytes(scatter_dp(d), n_classes, ring);
    const int rc = with_rows(x_dtype, s.X, [&](auto* Xr) {
      using T = row_t<decltype(Xr)>;
      auto kernel = ring ? class_scatter_kernel<T, true> : class_scatter_kernel<T, false>;
      return launch_smem(kernel, grid, tile_threads(ring), smem, ctx->stream, Xr, s.rows, d, ldx, s.y, s.mask, keep,
                         n_classes, static_cast<const double*>(ctx->disc), ctx->disc_part);
    });
    if (rc != B2_OK) return rc;
    return launch_ordered_reduce(ctx, ctx->disc_part, kDaPart, grid, s.first, kDaHead, 0u, ctx->disc + kDaSums, d,
                                 kDaHead, kMaxD);
  });
}

}  // namespace b2
