// b2_ptx.cuh -- PTX wrappers shared by the TMA / mbarrier pipelines (gram_tc.cu, gram_narrow.cu).
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

}  // namespace b2
