// b2_ptx.cuh -- PTX wrappers shared by the TMA / mbarrier pipelines (gram_tc.cu, gram_narrow.cu, score.cu), and the
// bulk-copy ring (ring_init, ring_produce) of the streaming kernels gram_narrow_kernel, score_tma_kernel,
// score_narrow_kernel, grad_tma_kernel and grad_narrow_kernel, and of the fp64 tile passes' TileRing (b2_dmma.cuh:
// glm_kernel, loo_kernel, score_std_kernel).
#pragma once
#include <cuda_bf16.h>
#include <stdint.h>

namespace b2 {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ uint64_t globaltimer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}
// Wait with a hardware suspend hint (the thread sleeps inside try_wait and is woken by the arrive, so
// waiting warps do not burn issue slots).  Bounded: a protocol bug must end in a trap (a clean launch
// failure), never in a hung GPU.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity, uint32_t hint_ns = 20000u) {
  uint32_t done = 0;
  uint64_t t0 = 0;
  while (true) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(bar), "r"(parity), "r"(hint_ns)
        : "memory");
    if (done) break;
    const uint64_t now = globaltimer_ns();
    if (t0 == 0) t0 = now;
    else if (now - t0 > 4000000000ull) __trap();
  }
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

__device__ __forceinline__ float ld_shared_f32(uint32_t addr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ uint32_t ld_shared_u8(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}
// one element of the raw tile as fp32 (T = float: 4-byte load; T = bf16: 2-byte load, widen)
template <typename T>
__device__ __forceinline__ float raw_ld_shared(uint32_t addr);
template <>
__device__ __forceinline__ float raw_ld_shared<float>(uint32_t addr) { return ld_shared_f32(addr); }
template <>
__device__ __forceinline__ float raw_ld_shared<__nv_bfloat16>(uint32_t addr) {
  unsigned short h;
  asm volatile("ld.shared.u16 %0, [%1];" : "=h"(h) : "r"(addr));
  return __uint_as_float(((uint32_t)h) << 16);
}
template <typename T>
__device__ __forceinline__ float raw_ld_global(const T* p);
template <>
__device__ __forceinline__ float raw_ld_global<float>(const float* p) { return __ldg(p); }
template <>
__device__ __forceinline__ float raw_ld_global<__nv_bfloat16>(const __nv_bfloat16* p) {
  return __bfloat162float(*p);
}

// ---- shared-memory row loads ---------------------------------------------------------------
__device__ __forceinline__ void lds_v4(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void lds_v2(uint32_t addr, uint32_t (&r)[2]) {
  asm volatile("ld.shared.v2.b32 {%0, %1}, [%2];" : "=r"(r[0]), "=r"(r[1]) : "r"(addr));
}
__device__ __forceinline__ uint32_t lds_b32(uint32_t addr) {
  uint32_t r;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(r) : "r"(addr));
  return r;
}
__device__ __forceinline__ uint32_t lds_u16(uint32_t addr) {
  unsigned short h;
  asm volatile("ld.shared.u16 %0, [%1];" : "=h"(h) : "r"(addr));
  return h;
}

// NV consecutive values of one row, vector loads (the row pitch and `addr` are multiples of the load size)
template <typename T, int NV>
__device__ __forceinline__ void ld_vals_vec(uint32_t addr, float (&v)[NV]) {
  static_assert(NV == 1 || NV == 2 || NV == 4 || NV == 8 || NV == 16, "power-of-two group sizes only");
  if constexpr (sizeof(T) == 4) {
    if constexpr (NV >= 4) {
#pragma unroll
      for (int q = 0; q < NV / 4; ++q) {
        uint32_t r[4];
        lds_v4(addr + 16 * q, r);
#pragma unroll
        for (int k = 0; k < 4; ++k) v[4 * q + k] = __uint_as_float(r[k]);
      }
    } else if constexpr (NV == 2) {
      uint32_t r[2];
      lds_v2(addr, r);
      v[0] = __uint_as_float(r[0]); v[1] = __uint_as_float(r[1]);
    } else {
      v[0] = __uint_as_float(lds_b32(addr));
    }
  } else {   // bf16: two values per 32-bit word, element 0 in the low half
    if constexpr (NV >= 8) {
#pragma unroll
      for (int q = 0; q < NV / 8; ++q) {
        uint32_t r[4];
        lds_v4(addr + 16 * q, r);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          v[8 * q + 2 * k] = __uint_as_float(r[k] << 16);
          v[8 * q + 2 * k + 1] = __uint_as_float(r[k] & 0xffff0000u);
        }
      }
    } else if constexpr (NV == 4) {
      uint32_t r[2];
      lds_v2(addr, r);
#pragma unroll
      for (int k = 0; k < 2; ++k) { v[2 * k] = __uint_as_float(r[k] << 16); v[2 * k + 1] = __uint_as_float(r[k] & 0xffff0000u); }
    } else if constexpr (NV == 2) {
      const uint32_t r = lds_b32(addr);
      v[0] = __uint_as_float(r << 16); v[1] = __uint_as_float(r & 0xffff0000u);
    } else {
      v[0] = __uint_as_float(lds_u16(addr) << 16);
    }
  }
}

// NV values starting at feature `start` of a row with runtime feature count d (zero beyond d)
template <typename T, int NV>
__device__ __forceinline__ void ld_vals_any(uint32_t row_addr, int start, int d, float (&v)[NV]) {
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    const int j = start + k;
    v[k] = j < d ? raw_ld_shared<T>(row_addr + (uint32_t)j * sizeof(T)) : 0.f;
  }
}

// 1-D bulk copy global -> shared (TMA engine, no tensor map): 16-byte aligned addresses, size % 16 == 0
__device__ __forceinline__ void bulk_load_1d(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(bar), "l"(0x12F0000000000000ull)
      : "memory");
}

// ---- the bulk-copy ring: STAGES slots in shared memory, each with a full barrier (the producer's arrive plus the copied
// bytes) at bar_full + 8 s and an empty barrier (one arrive per consumer warp) at bar_empty + 8 s ------------------------
template <int STAGES>
__device__ __forceinline__ void ring_init(uint32_t bar_full, uint32_t bar_empty, uint32_t consumer_warps) {
  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(bar_full + 8 * s, 1);
      mbar_init(bar_empty + 8 * s, consumer_warps);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
}

// The loop of the one producer lane: tiles blockIdx.x, + gridDim.x, ... < n_tiles of tile_rows rows each.  Tile `it`
// goes to slot s = it % STAGES once the consumers have released it: tile_rows * row_bytes bytes of X at xs + s * x_stride,
// with has_y tile_rows floats of y at ys + s * y_stride, with has_mask tile_rows mask bytes at ms + s * m_stride.
template <int STAGES>
__device__ __forceinline__ void ring_produce(uint32_t bar_full, uint32_t bar_empty, int n_tiles, int tile_rows,
                                             const void* X, uint32_t row_bytes, uint32_t xs, uint32_t x_stride,
                                             bool has_y, const float* y, uint32_t ys, uint32_t y_stride,
                                             bool has_mask, const uint8_t* mask, uint32_t ms, uint32_t m_stride) {
  const uint32_t xb = (uint32_t)tile_rows * row_bytes, yb = (uint32_t)tile_rows * 4u, mb = (uint32_t)tile_rows;
  const uint32_t tx = xb + (has_y ? yb : 0u) + (has_mask ? mb : 0u);
  int it = 0;
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++it) {
    const int s = it % STAGES;
    if (it >= STAGES) mbar_wait(bar_empty + 8 * s, (uint32_t)((it / STAGES - 1) & 1));
    const uint32_t full = bar_full + 8 * s;
    mbar_expect_tx(full, tx);
    const int64_t row0 = (int64_t)tile * tile_rows;
    bulk_load_1d(xs + s * x_stride, reinterpret_cast<const char*>(X) + (size_t)row0 * row_bytes, xb, full);
    if (has_y) bulk_load_1d(ys + s * y_stride, y + row0, yb, full);
    if (has_mask) bulk_load_1d(ms + s * m_stride, mask + row0, mb, full);
  }
}

}  // namespace b2
