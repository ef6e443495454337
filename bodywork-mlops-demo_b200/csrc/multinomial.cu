// multinomial.cu -- the row passes of multinomial logistic regression (b2_multinomial_pass, b2_multinomial_line_search,
// b2_softmax_rows; DESIGN.md section 14).
//
// scikit-learn's Newton solver for HalfMultinomialLoss needs, at the K x (D + 1) coefficients [W b] of each iteration and
// with eta_k = z.[w_k b_k] per kept row (z = [x 1]), the softmax p_k = exp(eta_k - m) / s (m = max_k eta_k, s the sum of
// the exponentials), the loss log(s) + m - eta_y, the gradient g_k = p_k - [y = k] and the K (K + 1) / 2 class-pair
// blocks sum h_kl z z^T of the Hessian, h_kk = p_k (1 - p_k) and h_kl = -p_k p_l.  One pass per call over 32-row tiles:
//   (1) the tile -> shared memory as z = [x 1 0...] in fp64 from the stored value (exact), zero for rows not kept, and
//       each row's class (its index in the sorted classes, -1 for a kept row of no class, -2 for a row not kept);
//   (2) eta for the K classes (and, for the line search, deta = z.[s_k db_k]) on the fp64 tensor core: tile_product
//       against the resident [W b]^T (with the step beside it: at most 64 columns);
//   (3) per kept row, one warp per row and one lane per class: the softmax, the loss, g, and the row's counts;
//   (4) the gradient: thread j adds g_rk z_rj over the tile's rows in order;
//   (5) (Hessian) blockIdx.y selects one class pair k <= l: the rows scaled by h_kl, then the upper-block schedule
//       (b2_dmma.cuh) -- the 16 x 16 blocks on and above the diagonal of the (D + 1)^2 block, held in registers for the
//       whole launch;
//   (6) (ladder) the loss at eta + 2^-t deta, one step t per lane.
// The grid is row slices x class pairs (one pair per CTA: the accumulators of one block fill the registers).  Each CTA
// writes its sums at its pair's place in its slice's partial; one ordered reduce adds the slices in order for every pair
// at once, so two calls return identical sums and the launches per host block do not grow with K.
#include "b2_internal.cuh"
#include "b2_dmma.cuh"

namespace b2 {
namespace {

constexpr int kMnBlocks = (kMaxD + 1 + 15) / 16;   // 9 blocks of 16 columns of [x 1]
constexpr int kMnSB = (kMnBlocks * (kMnBlocks + 1) / 2 + kTileWarps - 1) / kTileWarps;   // 16 x 16 blocks per warp: 6
constexpr int kMnEp = 2 * kMaxClasses + 1;         // pitch of eta [row][eta_k, deta_k]
constexpr int kMnPp = kMaxClasses + 1;             // pitch of g [row][class]

__host__ __device__ inline int mn_dp(int d) { return (d + 1 + 15) & ~15; }   // columns of [x 1], padded to 16
__host__ __device__ inline int mn_cols(int n_classes, int mode) { return mode == kGlmLadder ? 2 * n_classes : n_classes; }
__host__ __device__ inline int mn_bpitch(int cols) { return 8 * ((cols + 7) / 8) + 4; }

// the entries of one row slice's partial (and of the reduced sums): the head, the gradient [K][d + 1], the pair blocks
// [P][dp][dp] (Hessian)
size_t mn_slice_doubles(int d, int n_classes, int mode) {
  if (mode == kGlmLadder) return kMnHead;
  const size_t n = kMnHead + (size_t)n_classes * (d + 1);
  if (mode != kGlmHessian) return n;
  const size_t dp = mn_dp(d);
  return n + (size_t)n_classes * (n_classes + 1) / 2 * dp * dp;
}

size_t mn_smem_bytes(int d, int n_classes, int mode, bool ring) {
  const int dp = mn_dp(d);
  const size_t tile = (size_t)kTileRows * tile_vpitch(dp);
  const size_t gacc = (size_t)(mode == kGlmGradient ? n_classes : 1) * dp;
  return tile_ring_bytes(ring, true) +
         sizeof(double) * (tile * (mode == kGlmHessian ? 2 : 1) + (size_t)dp * mn_bpitch(mn_cols(n_classes, mode)) +
                           kTileRows * (kMnEp + kMnPp + 1) + gacc + 2 * kTileWarps * 32) +
         sizeof(float) * kMaxClasses + sizeof(int) * (kTileRows + kUpperTable);
}

// the class pair (k, l), k <= l, of pair index p in row-major order
__device__ __forceinline__ void mn_pair(int p, int n_classes, int& k, int& l) {
  k = 0;
  while (p >= n_classes - k) { p -= n_classes - k; ++k; }
  l = k + p;
}

// MODE kGlmGradient: slice partial [head | gradient], one CTA per slice.  kGlmHessian: CTA (slice, pair (k, l)) writes
// the block of its pair; the diagonal pairs also the gradient of class k, pair 0 the head.  kGlmLadder: the loss at step
// t in head[t], t < n_steps.  Head: [loss, kept, no class, y not finite, correct, 0...].  op: ctx->mn_op (kMn* in
// b2_internal.cuh).
template <typename T, bool RING, int MODE>
__global__ void __launch_bounds__(kTileThreads, 1)
multinomial_kernel(const T* __restrict__ X, int64_t n, int d, int64_t ldx, const float* __restrict__ y,
                   const uint8_t* __restrict__ mask, int keep, int n_classes, const double* __restrict__ op,
                   int n_steps, int64_t slice_doubles, double* __restrict__ part) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  TileRing<T, RING, true> tiles{X, n, d, ldx, y, mask, keep, smem_u32(smem_raw)};
  const int K = n_classes, dp = mn_dp(d), zp = tile_vpitch(dp), nb = dp / 16, nsb = nb * (nb + 1) / 2;
  const int cols = mn_cols(K, MODE), bp = mn_bpitch(cols), ntc = (cols + 7) / 8;
  double* Zs = reinterpret_cast<double*>(smem_raw + tile_ring_bytes(RING, true));   // [row][zp]: z = [x 1 0...]
  double* HZs = Zs + (MODE == kGlmHessian ? kTileRows * zp : 0);                   // h_kl z
  double* Bs = HZs + kTileRows * zp;         // [dp][bp]: [W b]^T (and [S db]^T), zero padded
  double* eta = Bs + dp * bp;                // [row][kMnEp]: eta_k, then deta_k at K + k
  double* gs = eta + kTileRows * kMnEp;      // [row][kMnPp]: g (0 for rows not kept)
  double* hs = gs + kTileRows * kMnPp;       // [row]: h_kl (0 for rows not kept)
  double* gacc = hs + kTileRows;             // [K or 1][dp]: the gradient rows of the CTA
  double* lsum = gacc + (MODE == kGlmGradient ? K : 1) * dp;   // [warp][u][8] the scalar sums of the rows warp + 8 u
  double* red = lsum + kTileWarps * 32;      // [warp][32] the ladder's per-lane sums
  float* cls = reinterpret_cast<float*>(red + kTileWarps * 32);
  int* row_cls = reinterpret_cast<int*>(cls + kMaxClasses);
  int* sb = row_cls + kTileRows;             // the upper blocks' table
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g8 = lane >> 2, t4 = lane & 3;
  // this CTA's pair and its gradient rows [k0, k1)
  int pk = 0, pl = 0, k0 = 0, k1 = K;
  if constexpr (MODE == kGlmHessian) {
    mn_pair(blockIdx.y, K, pk, pl);
    k0 = pk;
    k1 = pk == pl ? pk + 1 : pk;
  }
  const bool head = blockIdx.y == 0;
  for (int t = tid; t < kTileWarps * 32; t += blockDim.x) { lsum[t] = 0.0; red[t] = 0.0; }
  for (int t = tid; t < (MODE == kGlmGradient ? K : 1) * dp; t += blockDim.x) gacc[t] = 0.0;
  for (int t = tid; t < kMaxClasses; t += blockDim.x) cls[t] = t < K ? (float)op[kMnClasses + t] : 0.f;
  for (int t = tid; t < dp * bp; t += blockDim.x) {
    const int i = t / bp, c = t - i * bp;
    double v = 0.0;
    if (i <= d && c < K) v = op[kMnCoef + c * (kMaxD + 1) + i];
    else if (i <= d && c < cols) v = op[kMnStep + (c - K) * (kMaxD + 1) + i];
    Bs[t] = v;
  }
  upper_blocks(sb, nb);
  const int64_t n_tiles = (n + kTileRows - 1) / kTileRows;
  tiles.start();
  double s_loss = 0.0;                       // kGlmLadder: lane t sums the loss at step t
  double acc[MODE == kGlmHessian ? kMnSB : 1][4][2] = {};
  if (!tiles.produce()) {
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
      // (1) the tile: z = [x 1 0...], zero for rows not kept, and the rows' classes
      tiles.load(tile * kTileRows, dp,
                 [&](int r, int j, bool kept, bool live, float x) {
                   Zs[r * zp + j] = live ? (double)x : (kept && j == d ? 1.0 : 0.0);
                 },
                 [&](int r, bool kept, double yr) {
                   row_cls[r] = kept ? class_of(cls, K, (float)yr) : -2;
                   if (kept && !isfinite(yr)) lsum[(warp * 4 + (r >> 3)) * 8 + 3] += 1.0;
                 });
      tile_consumer_sync();
      // (2) eta (and deta) on the tensor core
      {
        double z[1][kTileMT][2];
        tile_product(Zs, zp, Bs, bp, dp, ntc, z);
        if (warp < ntc) {
#pragma unroll
          for (int mt = 0; mt < kTileMT; ++mt) {
            const int r = 8 * mt + g8, c = 8 * warp + 2 * t4;
            eta[r * kMnEp + c] = z[0][mt][0];
            eta[r * kMnEp + c + 1] = z[0][mt][1];
          }
        }
      }
      tile_consumer_sync();
      // (3) the pointwise terms of the warp's rows r = warp + 8 u
#pragma unroll 1
      for (int u = 0; u < kTileRowsPerWarp; ++u) {
        const int r = warp + kTileWarps * u, k = row_cls[r];
        const bool kept = k != -2;
        const double* er = eta + r * kMnEp;
        if constexpr (MODE == kGlmLadder) {
          // lane t: the loss at eta + 2^-t deta over the classes in order, sum_exp_minus_max
          const double t = ldexp(1.0, -lane);
          double m = -INFINITY;
          for (int c = 0; c < K; ++c) m = fmax(m, er[c] + t * er[K + c]);
          double s = 0.0;
          for (int c = 0; c < K; ++c) s += exp((er[c] + t * er[K + c]) - m);
          double l = log(s) + m;
          if (k >= 0) l -= er[k] + t * er[K + k];
          s_loss += (kept && lane < n_steps) ? l : 0.0;
        } else {
          // lane c: class c
          const double e = lane < K ? er[lane] : -INFINITY;
          double m = e;
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
          const double x = lane < K ? exp(e - m) : 0.0;
          double s = x;
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
          const double p = x / s;
          const double g = p - (lane == k ? 1.0 : 0.0);
          gs[r * kMnPp + lane] = kept ? g : 0.0;
          if constexpr (MODE == kGlmHessian) {
            const double p_k = __shfl_sync(0xffffffffu, p, pk), p_l = __shfl_sync(0xffffffffu, p, pl);
            if (lane == 0) hs[r] = kept ? (pk == pl ? p_k * (1.0 - p_k) : -p_k * p_l) : 0.0;
          }
          const double ey = __shfl_sync(0xffffffffu, e, k < 0 ? 0 : k);
          const unsigned top = __ballot_sync(0xffffffffu, lane < K && e == m);
          if (head && lane == 0) {
            double* ls = lsum + (warp * 4 + u) * 8;
            const double l = log(s) + m - (k >= 0 ? ey : 0.0);
            ls[0] += kept ? l : 0.0;
            ls[1] += kept ? 1.0 : 0.0;
            ls[2] += k == -1 ? 1.0 : 0.0;
            ls[4] += (k >= 0 && top != 0u && __ffs(top) - 1 == k) ? 1.0 : 0.0;
          }
        }
      }
      if constexpr (MODE != kGlmLadder) {
        tile_consumer_sync();
        // (4) the gradient rows of the CTA, then (Hessian) the h_kl-scaled rows
        if (tid <= d) {
          for (int c = k0; c < k1; ++c) {
            double* gc = gacc + (MODE == kGlmGradient ? c : 0) * dp + tid;
            double a = *gc;
#pragma unroll 8
            for (int r = 0; r < kTileRows; ++r) a = fma(gs[r * kMnPp + c], Zs[r * zp + tid], a);
            *gc = a;
          }
        }
        if constexpr (MODE == kGlmHessian) {
          for (int t = tid; t < kTileRows * dp; t += kTileConsumers) {
            const int r = t / dp, j = t - r * dp;
            HZs[r * zp + j] = hs[r] * Zs[r * zp + j];
          }
          tile_consumer_sync();
          // (5) H_kl += (h_kl z)^T z over the tile's rows, the warp's blocks
          upper_accumulate(acc, sb, nsb, [&](int r, int c) { return HZs[r * zp + c]; }, Zs, zp, warp, g8, t4);
        }
      }
      tile_consumer_sync();
    }
  }
  // the CTA's sums in a fixed order: the lanes of a warp, then the warps in order
  double* out = part + (size_t)blockIdx.x * slice_doubles;
  if constexpr (MODE == kGlmLadder) {
    if (warp < kTileWarps) red[warp * 32 + lane] = s_loss;
  }
  __syncthreads();
  if (head && tid < kMnHead) {
    double v = 0.0;
    if constexpr (MODE == kGlmLadder) {
      for (int w = 0; w < kTileWarps; ++w) v += red[w * 32 + tid];
    } else if (tid < 5) {
      for (int q = 0; q < kTileWarps * 4; ++q) v += lsum[q * 8 + tid];
    }
    out[tid] = v;
  }
  if constexpr (MODE != kGlmLadder) {
    for (int t = tid; t < (k1 - k0) * (d + 1); t += blockDim.x) {
      const int c = t / (d + 1), j = t - c * (d + 1);
      out[kMnHead + (k0 + c) * (d + 1) + j] = gacc[(MODE == kGlmGradient ? k0 + c : 0) * dp + j];
    }
  }
  if constexpr (MODE == kGlmHessian) {
    double* blk = out + kMnHead + (size_t)K * (d + 1) + (size_t)blockIdx.y * dp * dp;
    // the entries no accumulator covers (below the diagonal blocks, and the lower 8 x 8 tile of each) are zero
    for (int t = tid; t < dp * dp; t += blockDim.x) {
      const int i = t / dp, j = t - i * dp, bi = i >> 4, bj = j >> 4;
      if (bi > bj || (bi == bj && (i & 15) >= 8 && (j & 15) < 8)) blk[t] = 0.0;
    }
    upper_store(acc, sb, nsb, blk, dp, warp, g8, t4);
  }
}

// the softmax of each row of an (n, K) fp64 array in place, the steps of sklearn.utils.extmath.softmax: x - max, exp,
// / the sum.  The sum runs in column order; numpy's row sum (8-way unrolled and pairwise from K = 8) may round
// differently, by an ulp or so.
__global__ void __launch_bounds__(256)
softmax_rows_kernel(double* __restrict__ v, int64_t n, int k) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; row < n; row += stride) {
    double* r = v + row * k;
    double m = r[0];
    for (int c = 1; c < k; ++c) m = fmax(m, r[c]);
    double s = 0.0;
    for (int c = 0; c < k; ++c) {
      const double e = exp(r[c] - m);
      r[c] = e;
      s += e;
    }
    for (int c = 0; c < k; ++c) r[c] /= s;
  }
}

int ensure_mn_part(b2_ctx* ctx, size_t doubles) {
  if (doubles <= ctx->mn_part_doubles) return B2_OK;
  if (ctx->mn_part != nullptr) cudaFree(ctx->mn_part);
  ctx->mn_part = nullptr;
  ctx->mn_part_doubles = 0;
  if (cudaMalloc(reinterpret_cast<void**>(&ctx->mn_part), sizeof(double) * doubles) != cudaSuccess) {
    cudaGetLastError();
    set_error("out of device memory for the per-CTA partials of the multinomial pass (%zu doubles)", doubles);
    return B2_E_CUDA;
  }
  ctx->mn_part_doubles = doubles;
  return B2_OK;
}

}  // namespace

size_t multinomial_sum_doubles(int d, int n_classes, int mode) { return mn_slice_doubles(d, n_classes, mode); }

// The rows [0, n) in split_ring_rows's launches: slices x pairs CTAs (Hessian: as many slices as fill the SMs once with
// the pairs, at least one; otherwise one CTA per SM), then one ordered reduce of every slice's partial into ctx->mn_sum
// (`first_block` overwrites, otherwise adds).
int launch_multinomial(b2_ctx* ctx, const void* X, int x_dtype, int64_t n, int d, int64_t ldx, const float* y,
                       const uint8_t* mask, int keep, int mode, int n_classes, int n_steps, bool first_block) {
  const int pairs = mode == kGlmHessian ? n_classes * (n_classes + 1) / 2 : 1;
  const size_t slice = mn_slice_doubles(d, n_classes, mode);
  return split_ring_rows(ctx, X, x_dtype, n, d, ldx, y, mask, kTileRows, first_block, [&](bool ring, const RowSpan& s) {
    const int per = ctx->sm_count / pairs;
    const int slices = tile_grid(s.rows, per > 0 ? per : 1, 1);
    if (int r = ensure_mn_part(ctx, (size_t)slices * slice)) return r;
    const uint32_t smem = (uint32_t)mn_smem_bytes(d, n_classes, mode, ring);
    const dim3 grid(slices, pairs);
    const int rc = with_rows(x_dtype, s.X, [&](auto* Xr) {
      using T = row_t<decltype(Xr)>;
      return with_int<kGlmGradient, kGlmHessian, kGlmLadder>(mode, [&](auto M) {
        constexpr int MODE = decltype(M)::value;
        auto kernel = ring ? multinomial_kernel<T, true, MODE> : multinomial_kernel<T, false, MODE>;
        B2_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        kernel<<<grid, tile_threads(ring), smem, ctx->stream>>>(Xr, s.rows, d, ldx, s.y, s.mask, keep, n_classes,
                                                                 static_cast<const double*>(ctx->mn_op), n_steps,
                                                                 (int64_t)slice, ctx->mn_part);
        B2_CUDA(cudaGetLastError());
        return B2_OK;
      });
    });
    if (rc != B2_OK) return rc;
    return launch_ordered_reduce(ctx, ctx->mn_part, (int)slice, slices, s.first, (int)slice, 0u, ctx->mn_sum);
  });
}

int launch_softmax_rows(b2_ctx* ctx, double* values, int64_t n, int k) {
  if (n == 0) return B2_OK;
  const int64_t want = (n + 255) / 256, cap = (int64_t)ctx->sm_count * 8;
  softmax_rows_kernel<<<(int)(want < cap ? want : cap), 256, 0, ctx->stream>>>(values, n, k);
  B2_CUDA(cudaGetLastError());
  ctx->launches += 1;
  return B2_OK;
}

}  // namespace b2
