// qda.cu -- the passes of QuadraticDiscriminantAnalysis (b2_class_scatters, b2_qda_decision; DESIGN.md section 17).
//
// Every solver of scikit-learn's QuadraticDiscriminantAnalysis needs, beyond the class counts and means (b2_class_sums),
// each class's own scatter S_k = sum over the kept rows of class k of (x - m_k)(x - m_k)^T.  One pass reads the rows once,
// in class order, so that a class holding most rows still spreads over every SM:
//   (1) the class-order step (three small launches that read only y and the mask): the kept rows of each class per
//       chunk of kQdChunk rows, an exclusive scan of those counts in class-major order that also cuts each class's rows
//       into work items of at most item_rows rows (item_rows from the total count: about two items per SM), and the
//       kept rows' indices written grouped by class, in row order within a class;
//   (2) one CTA per work item gathers 32 of its rows at a time through the index (the next 32 are loaded into registers
//       while the tensor core works on the current ones), forms u = x - m_k in fp64 from the exactly converted value,
//       and accumulates u^T u with the upper-block schedule (b2_dmma.cuh): 16 x 16 blocks on and above the diagonal,
//       each warp holding up to five for the whole item;
//   (3) one reduce adds each class's items in item order into its sum (`first` overwrites, otherwise adds), so repeated
//       calls are bit-identical.
// The indices are int32 over spans of at most kQdSpan rows, which bounds the scratch at 64 MB.
//
// The decision pass computes d_k = -1/2 |(x - m_k) W_k|^2 + c_k per row and class: 2 K D^2 flops against D * 4 bytes
// of row, fp64-compute bound like score_std_kernel.  The grid is (row slice, class); each CTA holds its W_k resident in
// shared memory and streams its slice through the tile ring, forms u = x - m_k in fp64, Z = U W_k on the fp64 tensor
// core (tile_product) and the row sums of Z o Z in a fixed order, and writes column k of the n x K decisions.  One small
// launch over the decision rows then gives the label (the first largest), the kept and correct rows against y and, for
// two classes, d_1 - d_0.
#include "b2_internal.cuh"
#include "b2_dmma.cuh"

namespace b2 {
namespace {

constexpr int kQsBlocks = kMaxD / 16;                                                      // 8 blocks of 16 columns
constexpr int kQsSB = (kQsBlocks * (kQsBlocks + 1) / 2 + kTileWarps - 1) / kTileWarps;   // 16 x 16 blocks per warp: 5
constexpr int kQsThreads = kTileConsumers;                                                 // 256: no producer warp
constexpr int kQsCols = kMaxD / 8;                                                         // columns per thread per gather
constexpr int kQdCntPitch = kMaxClasses + 3;                                               // per chunk: K classes, 3 counts
constexpr int kQdDecNT = kMaxD / 8 / kTileWarps;                                           // n-tiles per warp: 2

__host__ __device__ inline int qs_dp(int d) { return (d + 15) & ~15; }   // the features, padded to 16

// ---- (1) the class-order step ------------------------------------------------------------------------------------------
// the class of row r of the span: its index in the classes, -1 for a kept row of no class (NaN included), -2 not kept
__device__ __forceinline__ int row_class_of(const float* cls, int K, const float* __restrict__ y,
                                            const uint8_t* __restrict__ mask, int keep, int64_t r) {
  const bool kept = mask == nullptr || __ldg(mask + r) == (uint8_t)keep;
  return kept ? class_of(cls, K, __ldg(y + r)) : -2;
}

// cnt[chunk][k]: kept rows of class k in the chunk; at K, K + 1, K + 2 of kMaxClasses..: kept, no class, y not finite
__global__ void __launch_bounds__(256)
order_count_kernel(const float* __restrict__ y, const uint8_t* __restrict__ mask, int keep, int64_t n, int K,
                   const double* __restrict__ op, int* __restrict__ cnt) {
  __shared__ float cls[kMaxClasses];
  __shared__ int c[kQdCntPitch];
  for (int t = threadIdx.x; t < kQdCntPitch; t += blockDim.x) c[t] = 0;
  for (int t = threadIdx.x; t < kMaxClasses; t += blockDim.x) cls[t] = t < K ? (float)op[kQdClasses + t] : 0.f;
  __syncthreads();
  const int64_t r0 = (int64_t)blockIdx.x * kQdChunk, r1 = r0 + kQdChunk < n ? r0 + kQdChunk : n;
  for (int64_t r = r0 + threadIdx.x; r < r1; r += blockDim.x) {
    const int k = row_class_of(cls, K, y, mask, keep, r);
    if (k >= 0) atomicAdd(c + k, 1);
    if (k != -2) atomicAdd(c + kMaxClasses, 1);
    if (k == -1) atomicAdd(c + kMaxClasses + 1, 1);
    if (k != -2 && !isfinite(__ldg(y + r))) atomicAdd(c + kMaxClasses + 2, 1);
  }
  __syncthreads();
  for (int t = threadIdx.x; t < kQdCntPitch; t += blockDim.x) cnt[(size_t)blockIdx.x * kQdCntPitch + t] = c[t];
}

// One CTA: cnt[chunk][k] becomes the index-list position of the chunk's first row of class k (class-major exclusive
// scan), then the per-class totals, the span's counts and the work items (class, begin, end) of at most item_rows rows,
// class by class, into the header `hd` (kQdHd* below).
__global__ void __launch_bounds__(1024)
order_scan_kernel(int* __restrict__ cnt, int n_chunks, int K, int max_items, int items_per_sm_total,
                  int* __restrict__ hd) {
  __shared__ int wsum[32];
  __shared__ int base;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) base = 0;
  __syncthreads();
  for (int k = 0; k < K; ++k) {
    for (int c0 = 0; c0 < n_chunks; c0 += 1024) {
      const int c = c0 + tid;
      const int v = c < n_chunks ? cnt[(size_t)c * kQdCntPitch + k] : 0;
      int s = v;                                               // inclusive scan of the warp
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, s, o);
        if (lane >= o) s += t;
      }
      if (lane == 31) wsum[warp] = s;
      __syncthreads();
      if (warp == 0) {
        int w = wsum[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const int t = __shfl_up_sync(0xffffffffu, w, o);
          if (lane >= o) w += t;
        }
        wsum[lane] = w;                                        // inclusive over the warps
      }
      __syncthreads();
      const int excl = base + (warp > 0 ? wsum[warp - 1] : 0) + s - v;
      if (c < n_chunks) cnt[(size_t)c * kQdCntPitch + k] = excl;
      __syncthreads();
      if (tid == 0) base += wsum[31];
      __syncthreads();
    }
    if (tid == 0) hd[kQdHdStart + k + 1] = base;             // the end of class k's indices
  }
  // the span's three counts (whole numbers: any order)
  if (warp < 3) {
    int s = 0;
    for (int c = lane; c < n_chunks; c += 32) s += cnt[(size_t)c * kQdCntPitch + kMaxClasses + warp];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) hd[kQdHdCounts + warp] = s;
  }
  if (tid == 0) {
    hd[kQdHdStart] = 0;
    const int total = hd[kQdHdStart + K];
    int rows = (total + items_per_sm_total - 1) / items_per_sm_total;
    rows = rows < kTileRows ? kTileRows : (rows + kTileRows - 1) / kTileRows * kTileRows;
    int it = 0;
    for (int k = 0; k < K; ++k) {
      hd[kQdHdFirstItem + k] = it;
      for (int b = hd[kQdHdStart + k]; b < hd[kQdHdStart + k + 1] && it < max_items; b += rows, ++it) {
        const int e = b + rows < hd[kQdHdStart + k + 1] ? b + rows : hd[kQdHdStart + k + 1];
        hd[kQdHdItems + 3 * it] = k;
        hd[kQdHdItems + 3 * it + 1] = b;
        hd[kQdHdItems + 3 * it + 2] = e;
      }
    }
    hd[kQdHdFirstItem + K] = it;
    hd[kQdHdNItems] = it;
  }
}

// idx[pos]: the span's kept rows of a class, grouped by class in row order; pos from the scanned cnt.  One CTA per chunk,
// its rows in rounds of 256 in order, the warps of a round in order, the lanes of a warp in order.
__global__ void __launch_bounds__(256)
order_place_kernel(const float* __restrict__ y, const uint8_t* __restrict__ mask, int keep, int64_t n, int K,
                   const double* __restrict__ op, const int* __restrict__ cnt, int* __restrict__ idx) {
  __shared__ float cls[kMaxClasses];
  __shared__ int run[kMaxClasses];
  __shared__ int wc[8][kMaxClasses];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int t = tid; t < kMaxClasses; t += blockDim.x) {
    cls[t] = t < K ? (float)op[kQdClasses + t] : 0.f;
    run[t] = t < K ? cnt[(size_t)blockIdx.x * kQdCntPitch + t] : 0;
  }
  const int64_t r0 = (int64_t)blockIdx.x * kQdChunk, r1 = r0 + kQdChunk < n ? r0 + kQdChunk : n;
  for (int64_t rb = r0; rb < r1; rb += 256) {
    for (int t = tid; t < 8 * kMaxClasses; t += blockDim.x) wc[t / kMaxClasses][t % kMaxClasses] = 0;
    __syncthreads();
    const int64_t r = rb + tid;
    const int k = r < r1 ? row_class_of(cls, K, y, mask, keep, r) : -2;
    const unsigned same = __match_any_sync(0xffffffffu, k);
    const int rank = __popc(same & ((1u << lane) - 1u));
    if (k >= 0 && rank == 0) wc[warp][k] = __popc(same);
    __syncthreads();
    if (k >= 0) {
      int pos = run[k] + rank;
      for (int w = 0; w < warp; ++w) pos += wc[w][k];
      idx[pos] = (int)(r);
    }
    __syncthreads();
    if (tid < K) {
      int s = 0;
      for (int w = 0; w < 8; ++w) s += wc[w][tid];
      run[tid] += s;
    }
    __syncthreads();                       // wc is read above before the next round clears it
  }
}

// ---- (2) the scatter of each work item ---------------------------------------------------------------------------------
// shared memory: the gathered rows u [kTileRows][zp], the class mean [dp], the upper blocks' table
size_t scatters_smem_bytes(int dp) {
  return sizeof(double) * ((size_t)kTileRows * tile_vpitch(dp) + dp) + sizeof(int) * kUpperTable;
}

// Item blockIdx.x of the header (none past its item count): the upper blocks of sum u u^T over its rows into part[item]
// at i kMaxD + j.  X: the span.
template <typename T>
__global__ void __launch_bounds__(kQsThreads, 1)
class_scatters_kernel(const T* __restrict__ X, int d, int64_t ldx, const int* __restrict__ idx,
                      const int* __restrict__ hd, const double* __restrict__ op, double* __restrict__ part) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int item = blockIdx.x;
  if (item >= hd[kQdHdNItems]) return;
  const int k = hd[kQdHdItems + 3 * item], begin = hd[kQdHdItems + 3 * item + 1], end = hd[kQdHdItems + 3 * item + 2];
  const int dp = qs_dp(d), zp = tile_vpitch(dp), nb = dp / 16, nsb = nb * (nb + 1) / 2;
  double* Us = reinterpret_cast<double*>(smem_raw);   // [row][zp]: u = x - m_k
  double* Ms = Us + kTileRows * zp;                   // [dp] m_k, zero padded
  int* sb = reinterpret_cast<int*>(Ms + dp);          // the upper blocks' table
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g8 = lane >> 2, t4 = lane & 3;
  for (int t = tid; t < dp; t += blockDim.x) Ms[t] = t < d ? op[kQdMeans + k * kMaxD + t] : 0.0;
  upper_blocks(sb, nb);
  // thread (pr, pc) gathers row pr of each 32 and its columns pc + 8 q
  const int pr = tid >> 3, pc = tid & 7;
  float nx[kQsCols];
  auto fetch = [&](int g0) {
    const int p = g0 + pr;
    const bool live = p < end;
    const T* xr = X + (live ? (int64_t)__ldg(idx + p) : 0) * ldx;
#pragma unroll
    for (int q = 0; q < kQsCols; ++q) {
      const int j = pc + 8 * q;
      nx[q] = (live && j < d) ? ld_row_val<T>(xr + j) : 0.f;
    }
  };
  double acc[kQsSB][4][2] = {};            // the warp's blocks, held for the whole item
  __syncthreads();
  fetch(begin);
  for (int g0 = begin; g0 < end; g0 += kTileRows) {
    // u = x - m_k in fp64 from the exact value, zero past the item and the features
    const bool live = g0 + pr < end;
#pragma unroll
    for (int q = 0; q < kQsCols; ++q) {
      const int j = pc + 8 * q;
      if (j < dp) Us[pr * zp + j] = (live && j < d) ? (double)nx[q] - Ms[j] : 0.0;
    }
    __syncthreads();
    if (g0 + kTileRows < end) fetch(g0 + kTileRows);   // the next rows' loads are in flight during the products
    // S_k += u^T u over the 32 rows, the warp's blocks
    upper_accumulate(acc, sb, nsb, [&](int r, int c) { return Us[r * zp + c]; }, Us, zp, warp, g8, t4);
    __syncthreads();
  }
  upper_store(acc, sb, nsb, part + (size_t)item * kMaxD * kMaxD, kMaxD, warp, g8, t4);
}

// ---- (3) the ordered reduce -------------------------------------------------------------------------------------------
// sums[kQdSums + k kMaxD^2 + i kMaxD + j] (i <= j < d) = (first ? 0 : itself) + the items of class k in item order;
// block (0, 0) also adds the span's class counts and three counts at kQdCounts.  Grid (entry blocks, K).
__global__ void __launch_bounds__(256)
scatters_reduce_kernel(const double* __restrict__ part, const int* __restrict__ hd, int d, int first,
                       double* __restrict__ sums) {
  const int k = blockIdx.y, e = blockIdx.x * blockDim.x + threadIdx.x, i = e / d, j = e - i * d;
  if (blockIdx.x == 0 && k == 0 && threadIdx.x < kMaxClasses + 3) {
    const int t = threadIdx.x;
    const int v = t < kMaxClasses ? (t < gridDim.y ? hd[kQdHdStart + t + 1] - hd[kQdHdStart + t] : 0)
                                  : hd[kQdHdCounts + t - kMaxClasses];
    sums[kQdCounts + t] = (first ? 0.0 : sums[kQdCounts + t]) + (double)v;
  }
  if (e >= d * d || j < i) return;
  double* s = sums + kQdSums + (size_t)k * kMaxD * kMaxD + i * kMaxD + j;
  double a = first ? 0.0 : *s;
  for (int it = hd[kQdHdFirstItem + k]; it < hd[kQdHdFirstItem + k + 1]; ++it) a += part[(size_t)it * kMaxD * kMaxD + i * kMaxD + j];
  *s = a;
}

// ---- the decision pass ----------------------------------------------------------------------------------------------
size_t qda_smem_bytes(int dp, bool ring) {
  return tile_ring_bytes(ring, false) +
         sizeof(double) * ((size_t)dp * tile_bpitch(dp) + (size_t)kTileRows * tile_vpitch(dp) + kTileWarps * kTileRows +
                           kMaxD);
}

// decision[row][k] = -1/2 |(x - m_k) W_k|^2 + c_k for the rows [0, n) of the CTA's slice, k = blockIdx.y.  op: ctx->qda.
template <typename T, bool RING>
__global__ void __launch_bounds__(kTileThreads, 1)
qda_decision_kernel(const T* __restrict__ X, int64_t n, int d, int64_t ldx, int K, const double* __restrict__ op,
                    double* __restrict__ decision) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  TileRing<T, RING, false> tiles{X, n, d, ldx, nullptr, nullptr, 0, smem_u32(smem_raw)};
  const int k = blockIdx.y, dp = tile_dp(d), bp = tile_bpitch(dp), vp = tile_vpitch(dp), ntc = dp / 8;
  double* Bs = reinterpret_cast<double*>(smem_raw + tile_ring_bytes(RING, false));   // [dp][bp]: W_k, zero padded
  double* Vs = Bs + dp * bp;               // the tile: u = x - m_k
  double* qpart = Vs + kTileRows * vp;     // [warp][row] partial sums of z^2
  double* mean = qpart + kTileWarps * kTileRows;   // [kMaxD]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2;
  const double* W = op + kQdW + (size_t)k * d * d;   // pitch d
  for (int t = tid; t < dp * bp; t += blockDim.x) {
    const int i = t / bp, l = t - i * bp;
    Bs[t] = (i < d && l < d) ? W[i * d + l] : 0.0;
  }
  for (int t = tid; t < kMaxD; t += blockDim.x) mean[t] = t < d ? op[kQdMeans + k * kMaxD + t] : 0.0;
  const double ck = op[kQdConst + k];
  const int64_t n_tiles = (n + kTileRows - 1) / kTileRows;
  tiles.start();
  if (tiles.produce()) return;
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int64_t row0 = tile * kTileRows;
    tiles.load(row0, dp,
               [&](int r, int j, bool, bool live, float x) { Vs[r * vp + j] = live ? (double)x - mean[j] : 0.0; },
               [](int, bool, double) {});
    tile_consumer_sync();
    double z[kQdDecNT][kTileMT][2];
    tile_product(Vs, vp, Bs, bp, dp, ntc, z);
    double qp[kTileMT];
#pragma unroll
    for (int mt = 0; mt < kTileMT; ++mt) {
      qp[mt] = 0.0;
#pragma unroll
      for (int u = 0; u < kQdDecNT; ++u) {   // z is 0 past the n-tiles
        qp[mt] = fma(z[u][mt][0], z[u][mt][0], qp[mt]);
        qp[mt] = fma(z[u][mt][1], z[u][mt][1], qp[mt]);
      }
      double v = qp[mt];
      v += __shfl_xor_sync(0xffffffffu, v, 1);
      v += __shfl_xor_sync(0xffffffffu, v, 2);
      if ((lane & 3) == 0) qpart[warp * kTileRows + 8 * mt + g] = v;
    }
    tile_consumer_sync();
    if (tid < kTileRows && row0 + tid < n) {
      double q = 0.0;
      for (int w = 0; w < kTileWarps; ++w) q += qpart[w * kTileRows + tid];
      decision[(row0 + tid) * K + k] = -0.5 * q + ck;
    }
    tile_consumer_sync();
  }
}

// Per row of the decisions [n][K]: label = classes[the first largest], diff = d_1 - d_0 (K = 2), each if not null; with y,
// the kept rows and those whose y equals the label added to cnt[0], cnt[1].
__global__ void __launch_bounds__(256)
qda_label_kernel(const double* __restrict__ decision, int64_t n, int K, const double* __restrict__ op,
                 const float* __restrict__ y, const uint8_t* __restrict__ mask, int keep, float* __restrict__ label,
                 double* __restrict__ diff, unsigned long long* __restrict__ cnt) {
  __shared__ float cls[kMaxClasses];
  for (int t = threadIdx.x; t < kMaxClasses; t += blockDim.x) cls[t] = t < K ? (float)op[kQdClasses + t] : 0.f;
  __syncthreads();
  unsigned long long kept = 0, correct = 0;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += stride) {
    const double* dr = decision + r * K;
    int best = 0;
    double top = dr[0];
    for (int c = 1; c < K; ++c) {
      const double e = dr[c];
      best = e > top ? c : best;
      top = e > top ? e : top;
    }
    const float lab = cls[best];
    if (label != nullptr) label[r] = lab;
    if (diff != nullptr) diff[r] = dr[1] - dr[0];
    if (y != nullptr) {
      const bool k = mask == nullptr || __ldg(mask + r) == (uint8_t)keep;
      kept += k ? 1 : 0;
      correct += (k && __ldg(y + r) == lab) ? 1 : 0;
    }
  }
  if (y == nullptr) return;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    kept += __shfl_xor_sync(0xffffffffu, kept, o);
    correct += __shfl_xor_sync(0xffffffffu, correct, o);
  }
  if ((threadIdx.x & 31) == 0 && kept > 0) {   // whole counts: any order
    atomicAdd(cnt, kept);
    atomicAdd(cnt + 1, correct);
  }
}

}  // namespace

int qda_max_items(const b2_ctx* ctx) { return kQdItemsPerSm * ctx->sm_count + kMaxClasses; }

// The span [0, n) (n <= kQdSpan): the class order, the items' scatters and the ordered reduce into ctx->qda + kQdSums.
int launch_class_scatters(b2_ctx* ctx, const void* X, int x_dtype, int64_t n, int d, int64_t ldx, const float* y,
                          const uint8_t* mask, int keep, int n_classes, bool first_block) {
  const int n_chunks = (int)((n + kQdChunk - 1) / kQdChunk), max_items = qda_max_items(ctx);
  int* idx = static_cast<int*>(ctx->qda_scratch);
  int* cnt = ctx->qda_hd + kQdHdCnt;
  const double* op = ctx->qda;
  if (n_chunks > 0) {
    order_count_kernel<<<n_chunks, 256, 0, ctx->stream>>>(y, mask, keep, n, n_classes, op, cnt);
    B2_CUDA(cudaGetLastError());
  }
  order_scan_kernel<<<1, 1024, 0, ctx->stream>>>(cnt, n_chunks, n_classes, max_items,
                                                 kQdItemsPerSm * ctx->sm_count, ctx->qda_hd);
  B2_CUDA(cudaGetLastError());
  ctx->launches += 1 + (n_chunks > 0 ? 3 : 0);
  if (n_chunks > 0) {
    order_place_kernel<<<n_chunks, 256, 0, ctx->stream>>>(y, mask, keep, n, n_classes, op, cnt, idx);
    B2_CUDA(cudaGetLastError());
    const uint32_t smem = (uint32_t)scatters_smem_bytes(qs_dp(d));
    const int rc = with_rows(x_dtype, X, [&](auto* Xr) {
      using T = row_t<decltype(Xr)>;
      return launch_smem(class_scatters_kernel<T>, max_items, kQsThreads, smem, ctx->stream, Xr, d, ldx,
                         static_cast<const int*>(idx), static_cast<const int*>(ctx->qda_hd), op, ctx->qda_part);
    });
    if (rc != B2_OK) return rc;
  }
  const dim3 grid((unsigned)((d * d + 255) / 256), (unsigned)n_classes);
  scatters_reduce_kernel<<<grid, 256, 0, ctx->stream>>>(ctx->qda_part, ctx->qda_hd, d, first_block ? 1 : 0, ctx->qda);
  B2_CUDA(cudaGetLastError());
  ctx->launches += 1;
  return B2_OK;
}

// The decisions of the rows [0, n) into decision [n][n_classes] in the launches of split_ring_rows; then the labels,
// d_1 - d_0 and the counts into ctx->qda_hd + kQdHdCorrect (added to; the caller zeroes them), each if not null.
int launch_qda_decision(b2_ctx* ctx, const void* X, int x_dtype, int64_t n, int d, int64_t ldx, const float* y,
                        const uint8_t* mask, int keep, int n_classes, double* decision, float* label, double* diff) {
  const auto part = [&](bool ring, const RowSpan& s) {
    const int64_t n_tiles = (s.rows + kTileRows - 1) / kTileRows;
    int64_t slices = ctx->sm_count / n_classes;        // one wave of (slice, class) CTAs
    slices = slices < 1 ? 1 : slices > n_tiles ? n_tiles : slices;
    const dim3 grid((unsigned)slices, (unsigned)n_classes);
    const uint32_t smem = (uint32_t)qda_smem_bytes(tile_dp(d), ring);
    const int rc = with_rows(x_dtype, s.X, [&](auto* Xr) {
      using T = row_t<decltype(Xr)>;
      auto kernel = ring ? qda_decision_kernel<T, true> : qda_decision_kernel<T, false>;
      B2_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
      kernel<<<grid, tile_threads(ring), smem, ctx->stream>>>(Xr, s.rows, d, ldx, n_classes,
                                                              static_cast<const double*>(ctx->qda),
                                                              decision + (size_t)s.r0 * n_classes);
      B2_CUDA(cudaGetLastError());
      return B2_OK;
    });
    if (rc != B2_OK) return rc;
    ctx->launches += 1;
    return B2_OK;
  };
  if (n == 0) return B2_OK;
  if (int r = split_ring_rows(ctx, X, x_dtype, n, d, ldx, nullptr, nullptr, kTileRows, false, part)) return r;
  if (label == nullptr && diff == nullptr && y == nullptr) return B2_OK;
  const int64_t want = (n + 2047) / 2048, cap = (int64_t)ctx->sm_count * 8;
  const int grid = (int)(want < cap ? want : cap);
  qda_label_kernel<<<grid, 256, 0, ctx->stream>>>(decision, n, n_classes, ctx->qda, y, mask, keep, label, diff,
                                                  reinterpret_cast<unsigned long long*>(ctx->qda_hd + kQdHdCorrect));
  B2_CUDA(cudaGetLastError());
  ctx->launches += 1;
  return B2_OK;
}

}  // namespace b2
