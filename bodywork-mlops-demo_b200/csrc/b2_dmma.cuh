// b2_dmma.cuh -- the device side shared by the fp64 tile passes: the fp64 tensor-core MMA, the per-element row load,
// the 32-row tile ring, its loader (step 1 of each pass), the product with an operand resident in shared memory
// (tile_product), and the upper-block schedule of the passes that sum a symmetric matrix.
//
// A pass runs kTileWarps consumer warps over the tiles blockIdx.x, + gridDim.x, ... of 32 rows.  In the ring flavour
// (rows [0, n), n a multiple of kTileRows, contiguous and 16-byte aligned, y too) one more warp's lane 0 runs
// ring_produce into kTileStages slots at the start of dynamic shared memory: the X stages, the y stages (HAS_Y), the
// full and empty barriers; the pass's doubles start tile_ring_bytes later, 16-byte aligned.  The direct flavour reads
// rows of any layout (stride ldx, fp32 or bf16, any alignment) from global memory and has no ring.
#pragma once
#include <cuda_bf16.h>

#include "b2_internal.cuh"
#include "b2_ptx.cuh"

namespace b2 {

__device__ __forceinline__ void dmma(double& c0, double& c1, double a, double b) {
  // fragments (PTX mma.m8n8k4.f64): A row = lane / 4, col = lane % 4; B row(k) = lane % 4, col(n) = lane / 4;
  // C row = lane / 4, cols = 2 (lane % 4) + {0, 1}
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
               : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}

template <typename T>
__device__ __forceinline__ float ld_row_val(const T* __restrict__ p);
template <>
__device__ __forceinline__ float ld_row_val<float>(const float* __restrict__ p) { return __ldg(p); }
template <>
__device__ __forceinline__ float ld_row_val<__nv_bfloat16>(const __nv_bfloat16* __restrict__ p) {
  return __bfloat162float(*p);
}

constexpr int kTileRows = 32;                            // rows per tile
constexpr int kTileMT = kTileRows / 8;                   // m-tiles of the DMMA per tile
constexpr int kTileWarps = 8;                            // consumer warps
constexpr int kTileRowsPerWarp = kTileRows / kTileWarps; // warp w holds the rows w + kTileWarps u
constexpr int kTileConsumers = 32 * kTileWarps;
constexpr int kTileThreads = kTileConsumers + 32;        // + the producer warp of the ring
constexpr int kTileStages = 3;
constexpr uint32_t kTileXStage = kTileRows * kMaxD * 4;  // 16 KB: 32 fp32 rows of 128 features
constexpr uint32_t kTileYStage = kTileRows * 4;
__host__ __device__ constexpr uint32_t tile_bar_offset(bool has_y) {
  return kTileStages * (kTileXStage + (has_y ? kTileYStage : 0u));
}
__host__ __device__ constexpr uint32_t tile_ring_bytes(bool ring, bool has_y) {   // where the doubles start
  return ring ? tile_bar_offset(has_y) + 2 * kTileStages * 8 + 16 : 0u;
}

// the features padded to 8, the tile's pitch and a resident operand's pitch, in doubles
__host__ __device__ inline int tile_dp(int d) { return (d + 7) & ~7; }
__host__ __device__ inline int tile_vpitch(int dp) { return dp + 4; }
__host__ __device__ inline int tile_bpitch(int dp) { return dp + 8; }

// CTAs of a launch over `rows` rows: one per tile up to ctas_per_sm per SM, and one without rows (it writes zero sums)
inline int tile_grid(int64_t rows, int sm_count, int ctas_per_sm) {
  const int64_t n_tiles = (rows + kTileRows - 1) / kTileRows, cap = (int64_t)sm_count * ctas_per_sm;
  const int grid = (int)(n_tiles < cap ? n_tiles : cap);
  return grid < 1 ? 1 : grid;
}
inline int tile_threads(bool ring) { return ring ? kTileThreads : kTileConsumers; }

// the consumer warps only (the producer is inside ring_produce)
__device__ __forceinline__ void tile_consumer_sync() {
  asm volatile("bar.sync 1, %0;" ::"r"(kTileConsumers) : "memory");
}

// The rows [0, n) of a tile pass: X (row pitch ldx), y (HAS_Y) and the mask (null: every row; else the rows with
// mask[row] == keep) as the kernel got them, and the ring's state.
template <typename T, bool RING, bool HAS_Y>
struct TileRing {
  const T* X;
  int64_t n;
  int d;
  int64_t ldx;
  const float* y;
  const uint8_t* mask;
  int keep;
  uint32_t sbase;                  // the dynamic shared memory
  int s = 0;                       // the slot of the next tile and its phase
  uint32_t phase = 0;
  int warp = (int)threadIdx.x >> 5;

  __device__ __forceinline__ uint32_t bar_full() const { return sbase + tile_bar_offset(HAS_Y); }
  __device__ __forceinline__ uint32_t bar_empty() const { return bar_full() + 8 * kTileStages; }

  // the ring's barriers, then a block barrier: call it after the pass has set up its shared memory
  __device__ __forceinline__ void start() const {
    if constexpr (RING) ring_init<kTileStages>(bar_full(), bar_empty(), kTileWarps);   // includes a block barrier
    else __syncthreads();
  }

  // true on the producer warp of the ring flavour, after its lane 0 has streamed the CTA's tiles of X (and y)
  __device__ __forceinline__ bool produce() const {
    if (!RING || warp != kTileWarps) return false;
    if ((threadIdx.x & 31) == 0)
      ring_produce<kTileStages>(bar_full(), bar_empty(), (int)((n + kTileRows - 1) / kTileRows), kTileRows, X,
                                (uint32_t)(d * sizeof(T)), sbase, kTileXStage, HAS_Y, y,
                                sbase + kTileStages * kTileXStage, kTileYStage, false, nullptr, 0u, 0u);
    return true;
  }

  // (1) the tile at row0 for the calling consumer warp.  For each of its rows r = warp + kTileWarps u: use[u] (the row
  // is in [0, n) and kept); store_x(r, j, use[u], live, x) for every j < dp, live = use[u] && j < d, x the stored value
  // as fp32 where live and 0 elsewhere (the store widens it to fp64 under `live`, once); with HAS_Y, store_y(r, use[u],
  // y) on lane 0, y the stored value in fp64 for a kept row and 0 otherwise.  The ring flavour reads the mask before it
  // waits for the slot, and releases the slot once the warp's stores are done.  No barrier beyond the warp: the pass
  // syncs what it shares.  This form hands use[] back in registers, its direct flavour unrolled over the warp's rows.
  template <typename StoreX, typename StoreY>
  __device__ __forceinline__ void load(int64_t row0, int dp, bool (&use)[kTileRowsPerWarp], StoreX&& store_x,
                                       StoreY&& store_y) {
    load_rows<true>(row0, dp, use, store_x, store_y);
  }
  // The same for a pass that keeps no row flag after the load: its direct flavour loops over the warp's rows rolled,
  // which keeps the row's registers free for the pass's products.
  template <typename StoreX, typename StoreY>
  __device__ __forceinline__ void load(int64_t row0, int dp, StoreX&& store_x, StoreY&& store_y) {
    bool use[kTileRowsPerWarp];
    load_rows<false>(row0, dp, use, store_x, store_y);
  }

 private:
  template <bool KEEP_USE, typename StoreX, typename StoreY>
  __device__ __forceinline__ void load_rows(int64_t row0, int dp, bool (&use)[kTileRowsPerWarp], StoreX& store_x,
                                            StoreY& store_y) {
    const int lane = threadIdx.x & 31;
    if constexpr (RING) {
#pragma unroll
      for (int u = 0; u < kTileRowsPerWarp; ++u)   // the mask comes from global memory, before the wait
        use[u] = mask == nullptr || __ldg(mask + row0 + warp + kTileWarps * u) == (uint8_t)keep;
      mbar_wait(bar_full() + 8 * s, phase);
      const uint32_t xs = sbase + s * kTileXStage, ys = sbase + kTileStages * kTileXStage + s * kTileYStage;
#pragma unroll
      for (int u = 0; u < kTileRowsPerWarp; ++u) {
        const int r = warp + kTileWarps * u;
        const uint32_t xr = xs + (uint32_t)(r * d) * (uint32_t)sizeof(T);
        for (int j = lane; j < dp; j += 32) {
          const bool live = use[u] && j < d;
          const float x = live ? raw_ld_shared<T>(xr + (uint32_t)j * (uint32_t)sizeof(T)) : 0.f;
          store_x(r, j, use[u], live, x);
        }
        if (HAS_Y && lane == 0) store_y(r, use[u], use[u] ? (double)ld_shared_f32(ys + 4u * (uint32_t)r) : 0.0);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_empty() + 8 * s);      // the slot is converted: the producer may refill it
      if (++s == kTileStages) { s = 0; phase ^= 1u; }
    } else {
      auto row_of = [&](int r, bool& kept) {                   // row r from global memory; kept: in [0, n) and kept
        const int64_t row = row0 + r;
        kept = row < n && (mask == nullptr || __ldg(mask + row) == (uint8_t)keep);
        const T* xr = X + row * ldx;
        for (int j = lane; j < dp; j += 32) {
          const bool live = kept && j < d;
          const float x = live ? ld_row_val<T>(xr + j) : 0.f;
          store_x(r, j, kept, live, x);
        }
        if (HAS_Y && lane == 0) store_y(r, kept, kept ? (double)__ldg(y + row) : 0.0);
      };
      if constexpr (KEEP_USE) {
#pragma unroll
        for (int u = 0; u < kTileRowsPerWarp; ++u) row_of(warp + kTileWarps * u, use[u]);
      } else {
        for (int r = warp; r < kTileRows; r += kTileWarps) row_of(r, use[0]);
      }
    }
  }
};

// (2) Z = V B on the fp64 tensor core (mma.sync m8n8k4 f64) for one tile: V the kTileRows x dp tile (pitch vp), B the
// dp x 8 ntc operand resident in shared memory (pitch bp).  Warp w takes the n-tiles w, w + kTileWarps, ... < ntc, at
// most NT of them, and all m-tiles: z[u][mt] is the C fragment of n-tile w + kTileWarps u, m-tile mt (0 past ntc).
template <int NT>
__device__ __forceinline__ void tile_product(const double* Vs, int vp, const double* Bs, int bp, int dp, int ntc,
                                             double (&z)[NT][kTileMT][2]) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t4 = lane & 3;
#pragma unroll
  for (int u = 0; u < NT; ++u) {
#pragma unroll
    for (int mt = 0; mt < kTileMT; ++mt) { z[u][mt][0] = 0.0; z[u][mt][1] = 0.0; }
    const int nt = warp + kTileWarps * u;
    if (nt < ntc) {
      for (int ks = 0; ks < dp / 4; ++ks) {
        const double b = Bs[(4 * ks + t4) * bp + 8 * nt + g];
        double a[kTileMT];
#pragma unroll
        for (int mt = 0; mt < kTileMT; ++mt) a[mt] = Vs[(8 * mt + g) * vp + 4 * ks + t4];
#pragma unroll
        for (int mt = 0; mt < kTileMT; ++mt) dmma(z[u][mt][0], z[u][mt][1], a[mt], b);
      }
    }
  }
}

// The upper-block schedule of the symmetric dp x dp fp64 sums (dp a multiple of 16): the Hessians of glm_kernel,
// multinomial_kernel and svm_kernel, the scatters of class_scatter_kernel and class_scatters_kernel.  A CTA writes
// every entry of the 16 x 16 blocks on and above the diagonal except the 8 x 8 tile below the diagonal of a diagonal
// block: the upper triangle i <= j, which the host mirrors (unpack_upper in b2_api.cu).  Consumer warp w holds blocks
// w, w + kTileWarps, ... in acc[u][q] for the whole launch, q the 8 x 8 tile at rows 8 (q >> 1), columns 8 (q & 1).
constexpr int kUpperTable = 96;   // ints of shared memory for the block table: rows at [0, 48), columns at [48, 96)

// the table of the nb (nb + 1) / 2 blocks on and above the diagonal (nb <= 9), row-major; thread 0 writes it, so the
// caller's next block barrier publishes it
__device__ __forceinline__ void upper_blocks(int* sb, int nb) {
  if (threadIdx.x != 0) return;
  int k = 0;
  for (int i = 0; i < nb; ++i)
    for (int j = i; j < nb; ++j, ++k) { sb[k] = i; sb[kUpperTable / 2 + k] = j; }
}

// acc += A^T B over the 32 rows of a tile for the calling warp's blocks: A[r][c] = load_a(r, c), B the tile at Bs
// (pitch zp).  Four DMMAs per 2 + 2 fragment loads, three on a diagonal block.  warp, g8 = lane / 4 and t4 = lane % 4
// are the calling thread's, as the kernel already holds them.
template <int SB, typename LoadA>
__device__ __forceinline__ void upper_accumulate(double (&acc)[SB][4][2], const int* sb, int nsb, LoadA&& load_a,
                                                 const double* Bs, int zp, int warp, int g8, int t4) {
#pragma unroll
  for (int u = 0; u < SB; ++u) {
    const int b = warp + kTileWarps * u;
    if (b < nsb) {                               // warp-uniform
      const int bi = sb[b], bj = sb[kUpperTable / 2 + b], ci = 16 * bi + g8, cj = 16 * bj + g8;
      const bool diag = bi == bj;
#pragma unroll
      for (int ks = 0; ks < kTileRows / 4; ++ks) {
        const int r = 4 * ks + t4;
        const double a0 = load_a(r, ci), a1 = load_a(r, ci + 8);
        const double b0 = Bs[r * zp + cj], b1 = Bs[r * zp + cj + 8];
        dmma(acc[u][0][0], acc[u][0][1], a0, b0);
        dmma(acc[u][1][0], acc[u][1][1], a0, b1);
        if (!diag) dmma(acc[u][2][0], acc[u][2][1], a1, b0);
        dmma(acc[u][3][0], acc[u][3][1], a1, b1);
      }
    }
  }
}

// the calling warp's blocks to out[i * pitch + j]; the producer warp of the ring holds none
template <int SB>
__device__ __forceinline__ void upper_store(const double (&acc)[SB][4][2], const int* sb, int nsb, double* out,
                                            int pitch, int warp, int g8, int t4) {
#pragma unroll
  for (int u = 0; u < SB; ++u) {
    const int b = warp + kTileWarps * u;
    if (warp < kTileWarps && b < nsb) {
      const int bi = sb[b], bj = sb[kUpperTable / 2 + b];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        if (q == 2 && bi == bj) continue;
        const int i = 16 * bi + 8 * (q >> 1) + g8, j = 16 * bj + 8 * (q & 1) + 2 * t4;
        out[i * pitch + j] = acc[u][q][0];
        out[i * pitch + j + 1] = acc[u][q][1];
      }
    }
  }
}

}  // namespace b2
