// classify.cu -- the row passes of the ridge classifier (b2_class_sums, b2_classify, b2_label_values; DESIGN.md
// section 12).  Its solve (solve_classes_kernel) lives in solve.cu beside the LDL^T it restates.
//
// scikit-learn's RidgeClassifier regresses the +-1 targets of LabelBinarizer(pos_label=1, neg_label=-1) on the rows:
// (Xc^T Xc + alpha I) W = Xc^T Yc.  The Gram gives Xc^T Xc; the right-hand sides need, per class k, the sum of the
// centred rows of the class and its count, which the class-sum pass gathers in one HBM-bound pass over 32-row tiles:
//   (1) the tile -> shared memory as x - c in fp64 from the stored value, and each row's class (its index in the sorted
//       classes, -1 for a kept row of no class, -2 for a row not kept);
//   (2) thread (h, j) adds column j of the rows 16 h .. 16 h + 15 in order into the class rows of its half.
// The classify pass computes eta = x W^T + b per row on the fp64 tensor core (tile_product with W resident in shared
// memory), then the decision, the label of the first largest eta and the rows it gets right.
// The rows take scoring's plan (plan_rows) through the tile ring of b2_dmma.cuh; each CTA writes its sums in a fixed
// order and the ordered reduce adds the CTAs in order, so two calls return identical sums.
#include "b2_internal.cuh"
#include "b2_dmma.cuh"

namespace b2 {
namespace {

// shared memory of the class-sum pass: the ring, the tile [kTileRows][vp], the two halves' class rows [2][K][dp], the
// centre, the classes, the rows' classes and the warps' counts [kTileWarps][K + 3]
size_t class_sums_smem_bytes(int dp, int n_classes, bool ring) {
  return tile_ring_bytes(ring, true) +
         sizeof(double) * ((size_t)kTileRows * tile_vpitch(dp) + 2 * (size_t)n_classes * dp + kMaxD +
                           kTileWarps * (kMaxClasses + 3)) +
         sizeof(float) * kMaxClasses + sizeof(int) * kTileRows;
}

// Per CTA: part[k (d + 1) + j] = sum over its kept rows of class k of x_j - c_j (j < d), part[k (d + 1) + d] = the rows
// of class k, then at K (d + 1): kept rows, kept rows of no class, kept rows with y not finite.  op: ctx->cls.
template <typename T, bool RING>
__global__ void __launch_bounds__(kTileThreads, 1)
class_sums_kernel(const T* __restrict__ X, int64_t n, int d, int64_t ldx, const float* __restrict__ y,
                  const uint8_t* __restrict__ mask, int keep, int n_classes, const double* __restrict__ op,
                  double* __restrict__ part) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  TileRing<T, RING, true> tiles{X, n, d, ldx, y, mask, keep, smem_u32(smem_raw)};
  const int dp = tile_dp(d), vp = tile_vpitch(dp), K = n_classes;
  double* Vs = reinterpret_cast<double*>(smem_raw + tile_ring_bytes(RING, true));   // [row][vp]: x - c
  double* acc = Vs + kTileRows * vp;       // [2][K][dp] the class rows of the two halves
  double* cv = acc + 2 * K * dp;           // [kMaxD] c
  double* cnt = cv + kMaxD;                // [warp][K + 3]: rows per class, kept, no class, y not finite
  float* cls = reinterpret_cast<float*>(cnt + kTileWarps * (kMaxClasses + 3));
  int* row_class = reinterpret_cast<int*>(cls + kMaxClasses);
  const int tid = threadIdx.x, warp = tid >> 5;
  for (int t = tid; t < 2 * K * dp; t += blockDim.x) acc[t] = 0.0;
  for (int t = tid; t < kTileWarps * (kMaxClasses + 3); t += blockDim.x) cnt[t] = 0.0;
  for (int t = tid; t < kMaxD; t += blockDim.x) cv[t] = t < d ? op[kClsCenter + t] : 0.0;
  for (int t = tid; t < kMaxClasses; t += blockDim.x) cls[t] = t < K ? (float)op[kClsClasses + t] : 0.f;
  const int64_t n_tiles = (n + kTileRows - 1) / kTileRows;
  tiles.start();
  if (!tiles.produce()) {
    const int j = tid & (kTileConsumers / 2 - 1), h = tid / (kTileConsumers / 2);   // column j of half h
    double* my = acc + h * K * dp + j;
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
      // (1) the tile and the rows' classes; lane 0 of each warp counts its own rows
      tiles.load(tile * kTileRows, dp,
                 [&](int r, int jj, bool, bool live, float x) { Vs[r * vp + jj] = live ? (double)x - cv[jj] : 0.0; },
                 [&](int r, bool kept, double yr) {
                   const int k = kept ? class_of(cls, K, (float)yr) : -2;
                   row_class[r] = k;
                   double* c = cnt + warp * (kMaxClasses + 3);
                   if (k >= 0) c[k] += 1.0;
                   c[kMaxClasses] += kept ? 1.0 : 0.0;
                   c[kMaxClasses + 1] += k == -1 ? 1.0 : 0.0;
                   c[kMaxClasses + 2] += (kept && !isfinite(yr)) ? 1.0 : 0.0;
                 });
      tile_consumer_sync();
      // (2) the half's rows in order into their classes
      if (j < d) {
#pragma unroll 4
        for (int r = 16 * h; r < 16 * h + 16; ++r) {
          const int k = row_class[r];
          if (k >= 0) my[k * dp] += Vs[r * vp + j];
        }
      }
      tile_consumer_sync();
    }
  }
  __syncthreads();
  // the CTA's sums: the two halves, then the warps' counts in warp order
  double* out = part + (size_t)blockIdx.x * kClsPart;
  for (int t = tid; t < K * (d + 1); t += blockDim.x) {
    const int k = t / (d + 1), jj = t - k * (d + 1);
    double v = 0.0;
    if (jj < d) {
      v = acc[k * dp + jj] + acc[(K + k) * dp + jj];
    } else {
      for (int w = 0; w < kTileWarps; ++w) v += cnt[w * (kMaxClasses + 3) + k];
    }
    out[t] = v;
  }
  if (tid < 3) {
    double v = 0.0;
    for (int w = 0; w < kTileWarps; ++w) v += cnt[w * (kMaxClasses + 3) + kMaxClasses + tid];
    out[K * (d + 1) + tid] = v;
  }
}

// shared memory of the classify pass: the ring, the tile [kTileRows][vp], W^T [dp][bp], eta [kTileRows][kMaxClasses + 1],
// b, the classes
__host__ __device__ inline int classify_bpitch(int n_targets) { return 8 * ((n_targets + 7) / 8) + 4; }
size_t classify_smem_bytes(int dp, int n_targets, bool ring) {
  return tile_ring_bytes(ring, false) +
         sizeof(double) * ((size_t)kTileRows * tile_vpitch(dp) + (size_t)dp * classify_bpitch(n_targets) +
                           kTileRows * (kMaxClasses + 1) + kMaxClasses) +
         sizeof(float) * kMaxClasses;
}

// eta_t = x.w_t + b_t for t < T per row in fp64.  Outputs, each optional: decision [n][T]; label: classes[argmax_t eta_t]
// (the first largest), for T = 1 classes[1] where eta > 0 and classes[0] otherwise; with y, per CTA part[0] = kept rows
// and part[1] = kept rows whose y equals the label.  op: ctx->cls (W at kClsCoef, pitch kMaxD, b at kClsIntercept).
template <typename T, bool RING>
__global__ void __launch_bounds__(kTileThreads, 1)
classify_kernel(const T* __restrict__ X, int64_t n, int d, int64_t ldx, const float* __restrict__ y,
                const uint8_t* __restrict__ mask, int keep, int n_targets, const double* __restrict__ op,
                double* __restrict__ decision, float* __restrict__ label, double* __restrict__ part) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  TileRing<T, RING, false> tiles{X, n, d, ldx, nullptr, nullptr, 0, smem_u32(smem_raw)};   // every row is scored
  const int dp = tile_dp(d), vp = tile_vpitch(dp), nt_t = n_targets, bp = classify_bpitch(nt_t), ntc = (nt_t + 7) / 8;
  constexpr int ep = kMaxClasses + 1;
  double* Vs = reinterpret_cast<double*>(smem_raw + tile_ring_bytes(RING, false));   // [row][vp]: x
  double* Bs = Vs + kTileRows * vp;        // [dp][bp]: W^T, zero padded
  double* eta = Bs + dp * bp;              // [row][ep]: x W^T
  double* bv = eta + kTileRows * ep;       // [kMaxClasses] b
  float* cls = reinterpret_cast<float*>(bv + kMaxClasses);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t4 = lane & 3;
  for (int t = tid; t < dp * bp; t += blockDim.x) {
    const int i = t / bp, c = t - i * bp;
    Bs[t] = (i < d && c < nt_t) ? op[kClsCoef + c * kMaxD + i] : 0.0;
  }
  for (int t = tid; t < kMaxClasses; t += blockDim.x) {
    bv[t] = t < nt_t ? op[kClsIntercept + t] : 0.0;
    cls[t] = t < (nt_t == 1 ? 2 : nt_t) ? (float)op[kClsClasses + t] : 0.f;
  }
  const int64_t n_tiles = (n + kTileRows - 1) / kTileRows;
  double kept_rows = 0.0, correct = 0.0;   // thread r < kTileRows: the rows r of the CTA's tiles
  tiles.start();
  if (!tiles.produce()) {
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
      const int64_t row0 = tile * kTileRows;
      tiles.load(row0, dp, [&](int r, int j, bool, bool live, float x) { Vs[r * vp + j] = live ? (double)x : 0.0; },
                 [](int, bool, double) {});
      tile_consumer_sync();
      double z[1][kTileMT][2];
      tile_product(Vs, vp, Bs, bp, dp, ntc, z);
      if (warp < ntc) {
#pragma unroll
        for (int mt = 0; mt < kTileMT; ++mt) {
          const int r = 8 * mt + g, c = 8 * warp + 2 * t4;
          eta[r * ep + c] = z[0][mt][0];
          eta[r * ep + c + 1] = z[0][mt][1];
        }
      }
      tile_consumer_sync();
      if (decision != nullptr) {
        for (int t = tid; t < kTileRows * nt_t; t += kTileConsumers) {
          const int r = t / nt_t, c = t - r * nt_t;
          if (row0 + r < n) decision[(row0 + r) * nt_t + c] = eta[r * ep + c] + bv[c];
        }
      }
      if (tid < kTileRows && row0 + tid < n) {
        const int64_t row = row0 + tid;
        int best = 0;
        double top = eta[tid * ep] + bv[0];
        for (int c = 1; c < nt_t; ++c) {
          const double e = eta[tid * ep + c] + bv[c];
          best = e > top ? c : best;
          top = e > top ? e : top;
        }
        const float lab = nt_t == 1 ? cls[top > 0.0 ? 1 : 0] : cls[best];
        if (label != nullptr) label[row] = lab;
        if (y != nullptr) {
          const bool kept = mask == nullptr || __ldg(mask + row) == (uint8_t)keep;
          kept_rows += kept ? 1.0 : 0.0;
          correct += (kept && __ldg(y + row) == lab) ? 1.0 : 0.0;
        }
      }
      tile_consumer_sync();
    }
  }
  // whole counts: the order of the adds does not matter
  if (warp == 0) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      kept_rows += __shfl_xor_sync(0xffffffffu, kept_rows, o);
      correct += __shfl_xor_sync(0xffffffffu, correct, o);
    }
    if (lane == 0 && part != nullptr) {
      part[(size_t)blockIdx.x * kClsPart] = kept_rows;
      part[(size_t)blockIdx.x * kClsPart + 1] = correct;
    }
  }
}

// One step of the label discovery: st[i] = the smallest order-preserving key of a finite kept y above st[i - 1] (any
// finite kept y for i = 0); nothing when st[i - 1] found none.  -0.0 is read as 0.0.
__global__ void __launch_bounds__(256)
label_next_kernel(const float* __restrict__ y, int64_t n, const uint8_t* __restrict__ mask, int keep, int i,
                  unsigned long long* __restrict__ st) {
  const unsigned long long none = ~0ull;
  const unsigned long long prev = i == 0 ? 0ull : st[i - 1];
  if (i > 0 && prev == none) return;
  unsigned long long kmin = none;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += stride) {
    if (mask != nullptr && __ldg(mask + r) != (uint8_t)keep) continue;
    const float v = __ldg(y + r) + 0.0f;   // -0 + 0 = +0
    if (!isfinite(v)) continue;
    const unsigned long long k = label_key(v);
    if ((i == 0 || k > prev) && k < kmin) kmin = k;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long a = __shfl_xor_sync(0xffffffffu, kmin, o);
    kmin = a < kmin ? a : kmin;
  }
  if ((threadIdx.x & 31) == 0 && kmin != none) atomicMin(st + i, kmin);
}

// two CTAs per SM where their shared memory fits (it overlaps one CTA's loads with the other's sums), one otherwise
int ctas_per_sm(size_t smem) { return 2 * (smem + 1024) <= 228 * 1024 ? 2 : 1; }

}  // namespace

int launch_class_sums(b2_ctx* ctx, const void* X, int x_dtype, int64_t n, int d, int64_t ldx, const float* y,
                      const uint8_t* mask, int keep, int n_classes, bool first_block) {
  return split_ring_rows(ctx, X, x_dtype, n, d, ldx, y, mask, kTileRows, first_block, [&](bool ring, const RowSpan& s) {
    const uint32_t smem = (uint32_t)class_sums_smem_bytes(tile_dp(d), n_classes, ring);
    const int grid = tile_grid(s.rows, ctx->sm_count, ctas_per_sm(smem));
    const int rc = with_rows(x_dtype, s.X, [&](auto* Xr) {
      using T = row_t<decltype(Xr)>;
      auto kernel = ring ? class_sums_kernel<T, true> : class_sums_kernel<T, false>;
      return launch_smem(kernel, grid, tile_threads(ring), smem, ctx->stream, Xr, s.rows, d, ldx, s.y, s.mask, keep,
                         n_classes, static_cast<const double*>(ctx->cls), ctx->glm_part);
    });
    if (rc != B2_OK) return rc;
    return launch_ordered_reduce(ctx, ctx->glm_part, kClsPart, grid, s.first, n_classes * (d + 1) + 3, 0u,
                                 ctx->cls + kClsSums);
  });
}

int launch_classify(b2_ctx* ctx, const void* X, int x_dtype, int64_t n, int d, int64_t ldx, const float* y,
                    const uint8_t* mask, int keep, int n_targets, double* decision, float* label, bool first_block) {
  return split_ring_rows(ctx, X, x_dtype, n, d, ldx, y, mask, kTileRows, first_block, [&](bool ring, const RowSpan& s) {
    const uint32_t smem = (uint32_t)classify_smem_bytes(tile_dp(d), n_targets, ring);
    const int grid = tile_grid(s.rows, ctx->sm_count, ctas_per_sm(smem));
    double* dec = decision != nullptr ? decision + (size_t)s.r0 * n_targets : nullptr;
    float* lab = label != nullptr ? label + s.r0 : nullptr;
    double* part = y != nullptr ? ctx->glm_part : nullptr;
    const int rc = with_rows(x_dtype, s.X, [&](auto* Xr) {
      using T = row_t<decltype(Xr)>;
      auto kernel = ring ? classify_kernel<T, true> : classify_kernel<T, false>;
      return launch_smem(kernel, grid, tile_threads(ring), smem, ctx->stream, Xr, s.rows, d, ldx, s.y, s.mask, keep,
                         n_targets, static_cast<const double*>(ctx->cls), dec, lab, part);
    });
    if (rc != B2_OK) return rc;
    if (y == nullptr) {
      ctx->launches += 1;
      return B2_OK;
    }
    return launch_ordered_reduce(ctx, ctx->glm_part, kClsPart, grid, s.first, 2, 0u, ctx->cls + kClsCounts);
  });
}

int launch_label_values(b2_ctx* ctx, const float* y, int64_t n, const uint8_t* mask, int keep, int max_values,
                        unsigned long long* st) {
  B2_CUDA(cudaMemsetAsync(st, 0xff, sizeof(unsigned long long) * (max_values + 1), ctx->stream));
  if (n == 0) return B2_OK;
  const int64_t want = (n + 2047) / 2048, cap = (int64_t)ctx->sm_count * 8;
  const int grid = (int)(want < cap ? want : cap);
  for (int i = 0; i <= max_values; ++i) {
    label_next_kernel<<<grid, 256, 0, ctx->stream>>>(y, n, mask, keep, i, st);
    B2_CUDA(cudaGetLastError());
  }
  ctx->launches += max_values + 1;
  return B2_OK;
}

}  // namespace b2
