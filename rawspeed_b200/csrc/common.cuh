// common.cuh -- shared device helpers for the rawspeed_b200 kernels (sm_90a).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace rsb200 {

__device__ __forceinline__ uint4 ldg_nc_v4(const void* p) {
  // streaming 128-bit read-only load, do not pollute L1
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}

__device__ __forceinline__ void stg_cs_v4(void* p, const uint4& v) {
  // streaming 128-bit store (evict-first)
  asm volatile("st.global.cs.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x),
               "r"(v.y), "r"(v.z), "r"(v.w)
               : "memory");
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// Explicit shared-window accesses for the hot loops.  The address operand is a
// 32-bit shared address held in a register plus a compile-time byte offset; the
// base comes from smem_base_opaque() ONCE per kernel: nvcc otherwise
// re-materialises the generic->shared conversion (S2R SR_CgaCtaId + LEA) next to
// every access inside the loops.
__device__ __forceinline__ uint32_t smem_base_opaque(const void* p) {
  uint32_t r;
  asm volatile("mov.u32 %0, %1;" : "=r"(r) : "r"(smem_u32(p)));
  return r;
}
template <int OFF = 0> __device__ __forceinline__ uint32_t lds_u16(uint32_t saddr) {
  uint16_t v;
  asm volatile("ld.shared.u16 %0, [%1+%2];" : "=h"(v) : "r"(saddr), "n"(OFF) : "memory");
  return v;
}
template <int OFF = 0> __device__ __forceinline__ uint32_t lds_u32(uint32_t saddr) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1+%2];" : "=r"(v) : "r"(saddr), "n"(OFF) : "memory");
  return v;
}
template <int OFF = 0> __device__ __forceinline__ void sts_u32(uint32_t saddr, uint32_t v) {
  asm volatile("st.shared.u32 [%0+%1], %2;" ::"r"(saddr), "n"(OFF), "r"(v) : "memory");
}
template <int OFF = 0> __device__ __forceinline__ void sts_u16(uint32_t saddr, uint32_t v) {
  asm volatile("st.shared.u16 [%0+%1], %2;" ::"r"(saddr), "n"(OFF), "h"((uint16_t)v) : "memory");
}
template <int OFF = 0> __device__ __forceinline__ uint32_t lds_u8(uint32_t saddr) {
  uint32_t v;
  asm volatile("ld.shared.u8 %0, [%1+%2];" : "=r"(v) : "r"(saddr), "n"(OFF) : "memory");
  return v;
}
template <int OFF = 0> __device__ __forceinline__ uint2 lds_v2(uint32_t saddr) {
  uint2 v;
  asm volatile("ld.shared.v2.u32 {%0,%1}, [%2+%3];" : "=r"(v.x), "=r"(v.y) : "r"(saddr), "n"(OFF) : "memory");
  return v;
}
template <int OFF = 0> __device__ __forceinline__ uint4 lds_v4(uint32_t saddr) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4+%5];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "r"(saddr), "n"(OFF)
               : "memory");
  return v;
}
template <int OFF = 0> __device__ __forceinline__ void sts_u8(uint32_t saddr, uint32_t v) {
  asm volatile("st.shared.u8 [%0+%1], %2;" ::"r"(saddr), "n"(OFF), "r"(v) : "memory");
}
template <int OFF = 0> __device__ __forceinline__ void sts_v2(uint32_t saddr, const uint2& v) {
  asm volatile("st.shared.v2.u32 [%0+%1], {%2,%3};" ::"r"(saddr), "n"(OFF), "r"(v.x), "r"(v.y) : "memory");
}
template <int OFF = 0> __device__ __forceinline__ void sts_v4(uint32_t saddr, const uint4& v) {
  asm volatile("st.shared.v4.u32 [%0+%1], {%2,%3,%4,%5};" ::"r"(saddr), "n"(OFF), "r"(v.x), "r"(v.y),
               "r"(v.z), "r"(v.w)
               : "memory");
}
// c + (a * b >> 32): with b a power of two this is "c + (a >> k)" on the FMA
// pipe (IMAD.HI), which the decode loops use to off-load the busier ALU pipe
__device__ __forceinline__ uint32_t mad_hi(uint32_t a, uint32_t b, uint32_t c) {
  uint32_t r;
  asm("mad.hi.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c));
  return r;
}

// PRMT in its generic form: nibble n of sel picks byte (sel_n & 7) of {b, a}; bit 3 of the nibble
// replicates that byte's sign bit instead (0x00 / 0xFF).  Only sel[15:0] is used.
__device__ __forceinline__ uint32_t prmt(uint32_t a, uint32_t b, uint32_t sel) {
  uint32_t r;
  asm("prmt.b32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(sel));
  return r;
}

// ---- mbarrier + 1-D bulk async copy (TMA unit, SASS: UBLKCP) ----
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(
                   smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t phase) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra.uni WAIT_DONE;\n\t"
      "bra.uni WAIT_LOOP;\n\t"
      "WAIT_DONE:\n\t"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(phase)
      : "memory");
}
// global -> shared bulk copy; dst/src 16-byte aligned, bytes % 16 == 0
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc,
                                         uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes "
      "[%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
      "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}

} // namespace rsb200
