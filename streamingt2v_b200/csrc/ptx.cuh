// Thin inline-PTX wrappers for sm_90a: mbarrier, TMA (cp.async.bulk.tensor), wgmma descriptors.
// Everything here is device-side and header-only.  No CUTLASS dependency.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200 {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ----------------------------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
// make generic-proxy smem writes visible to the async proxy (TMA / wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
// Wait that parks the thread in hardware (suspend-time hint, ns) instead of re-polling every few dozen cycles: for
// waits that are expected to be long and whose pollers would otherwise take issue slots from working warps.
__device__ __forceinline__ void mbar_wait_parked(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1, %2;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t}"
      ::"r"(smem_u32(bar)), "r"(parity), "r"(20000u)
      : "memory");
}

// ----------------------------------------------------------------------------------------------
// TMA tiled loads (global -> shared, completion on an mbarrier)
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                            int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], "
      "[%2];" ::"r"(smem_u32(smem)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, "
      "%6}], [%2];" ::"r"(smem_u32(smem)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_5d(void* smem, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2,
                                            int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, "
      "%6, %7}], [%2];" ::"r"(smem_u32(smem)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}

// TMA tiled store (shared -> global, bulk async group); out-of-bounds parts of the box are clipped by hardware
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* m, const void* smem, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.global.shared::cta.tile.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
          reinterpret_cast<uint64_t>(m)),
      "r"(smem_u32(smem)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_store_5d(const CUtensorMap* m, const void* smem, int c0, int c1, int c2, int c3,
                                             int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.global.shared::cta.tile.bulk_group [%0, {%2, %3, %4, %5, %6}], [%1];" ::"l"(
          reinterpret_cast<uint64_t>(m)),
      "r"(smem_u32(smem)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// wait until all committed bulk groups of this thread have finished READING shared memory
__device__ __forceinline__ void tma_store_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

__device__ __forceinline__ void named_bar_arrive(int id, int nthreads) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// ----------------------------------------------------------------------------------------------
// Descriptors
// ----------------------------------------------------------------------------------------------
// wgmma shared-memory matrix descriptor, K-major operand, 128-byte swizzle: rows of 64 x 16-bit (= 128 B), 8-row
// groups 1024 B apart (the dense tile a SWIZZLE_128B TMA box with a 64-element inner extent writes).  Stepping 16
// elements along K inside the swizzle atom adds 32 B (+2 in the address field).
__device__ __forceinline__ uint64_t smem_desc_k_sw128(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);  // start address  [0,14)
  d |= (uint64_t)1 << 16;                  // LBO (unused for swizzled K-major) = 1
  d |= (uint64_t)(1024 >> 4) << 32;        // SBO = 1024 B  [32,46)
  d |= (uint64_t)1 << 62;                  // layout type SWIZZLE_128B  [62,64)
  return d;
}
// MN-major operand, 128-byte swizzle: smem tile is [K rows][64 MN elements = 128 B]; 8-row (K) groups 1024 B apart.
__device__ __forceinline__ uint64_t smem_desc_mn_sw128(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)1 << 16;            // LBO: stride between 64-element MN atoms (single atom here)
  d |= (uint64_t)(1024 >> 4) << 32;  // SBO: stride between 8-deep K groups
  d |= (uint64_t)1 << 62;
  return d;
}
// K-major operand, 32-byte swizzle: rows of 16 x 16-bit (= 32 B, one k16 step), 8-row groups 256 B apart (the tile a
// SWIZZLE_32B TMA box with a 16-element inner extent writes).
__device__ __forceinline__ uint64_t smem_desc_k_sw32(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)1 << 16;           // LBO (unused for swizzled K-major) = 1
  d |= (uint64_t)(256 >> 4) << 32;  // SBO = 256 B
  d |= (uint64_t)3 << 62;           // layout type SWIZZLE_32B
  return d;
}
// MN-major operand, 32-byte swizzle: smem tile is [K rows][16 MN elements = 32 B]; 8-row (K) groups 256 B apart.
__device__ __forceinline__ uint64_t smem_desc_mn_sw32(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)1 << 16;           // LBO: stride between 16-element MN atoms (single atom here)
  d |= (uint64_t)(256 >> 4) << 32;  // SBO: stride between 8-deep K groups
  d |= (uint64_t)3 << 62;
  return d;
}

// ----------------------------------------------------------------------------------------------
// small math helpers
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ float silu_f(float x) { return x / (1.0f + __expf(-x)); }
// SiLU with approximate exp/reciprocal (rel err ~1e-6, far below bf16 rounding): ~5 instructions instead of ~20
__device__ __forceinline__ float silu_fast(float x) { return __fdividef(x, 1.0f + __expf(-x)); }
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float rcp_approx(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float gelu_f(float x) {  // exact (erf) GELU, matches torch F.gelu default
  return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f));
}
// GELU(x) = x * Phi(x) with erf via Abramowitz-Stegun 7.1.25 (|abs err| <= 2.5e-5, two orders below the bf16 output
// rounding): 2 MUFU + 10 FMA-pipe instructions, branch free.  erff's ~35 instructions made the GEGLU epilogue
// issue-bound.
//   gelu = h + |h| * erf(|x|/sqrt2),  h = x/2;  erf(z) = 1 - (a1 t + a2 t^2 + a3 t^3) exp(-z^2),  t = 1/(1 + p z)
__device__ __forceinline__ float gelu_fast(float x) {
  const float t = rcp_approx(fmaf(0.47047f * 0.70710678118654752440f, fabsf(x), 1.0f));
  float poly = fmaf(0.7478556f, t, -0.0958798f);
  poly = fmaf(poly, t, 0.3480242f);
  poly *= t;
  const float e = ex2_approx((x * x) * (-0.5f * 1.4426950408889634f));  // exp(-x^2/2)
  const float h = 0.5f * x;
  const float pe = poly * e;
  return fmaf(-fabsf(h), pe, h + fabsf(h));
}
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 t = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&t);
}
__device__ __forceinline__ float bf16_lo(uint32_t u) { return __uint_as_float(u << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t u) { return __uint_as_float(u & 0xFFFF0000u); }

}  // namespace b200
