// Inline-PTX wrappers for the Hopper (sm_90a) async machinery used by the tensor-core kernels:
// mbarrier, 1-D bulk copy (TMA), proxy fences, warpgroup MMA (wgmma) fences / groups, and the shared-memory matrix descriptor (K-major, no swizzle).
#pragma once
#include <cuda_fp16.h>
#include <stdint.h>

#include "wgmma_ops.cuh"

namespace mcvd {
namespace ptx {

// ---- PTX wrappers -----------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n\t}" ::"r"(bar),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done;
  do {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
  } while (!done);
}
// named barrier over a subset of the CTA's warps (ids 1..15; 0 is __syncthreads)
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}
// tiled tensor copy (TMA) of one box at element coordinates (c0, c1[, c2]); out-of-range elements are zero-filled
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const void* map, int c0, int c1, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
          dst),
      "l"(map), "r"(c0), "r"(c1), "r"(bar)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const void* map, int c0, int c1, int c2, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];" ::"r"(
          dst),
      "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(bar)
      : "memory");
}
// per-thread register budget of the executing warpgroup, lowered (registers go back to the CTA's pool) or raised
// (blocks until the pool holds them); every warp of the warpgroup executes it
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

// ---- warpgroup MMA ------------------------------------------------------------------------------
// wgmma_fence orders the warpgroup's register / shared-memory accesses before the next wgmma; commit closes a group of
// issued wgmmas; wait<N> blocks until at most N groups are still pending (their accumulators may then be read).
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keep the compiler from moving accumulator reads / writes across an asynchronous wgmma
__device__ __forceinline__ void reg_fence(float& r) { asm volatile("" : "+f"(r)::"memory"); }

// K-major, no-swizzle shared-memory matrix descriptor (wgmma "interleave" layout, cute::GMMA::GmmaDescriptor):
//   [0,14) start>>4 | [16,30) LBO>>4 (K-direction core-matrix stride) | [32,46) SBO>>4 (8-row group
//   stride) | [62,64) layout = 0 (no swizzle).  A core matrix is 8 rows x 16 bytes, rows 16 bytes apart.
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFFu);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;
  return d;
}
// descriptor with the start-address field advanced by `units16` (16-byte units); fields do not overlap
__device__ __forceinline__ uint64_t desc_add(uint64_t d, uint32_t units16) { return d + (uint64_t)units16; }

__device__ __forceinline__ uint32_t pack_half2(__half a, __half b) {
  return (uint32_t)__half_as_ushort(a) | ((uint32_t)__half_as_ushort(b) << 16);
}

// one elected lane of a converged warp
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t"
      "}"
      : "=r"(pred));
  return pred != 0;
}

// ---- cheap math for the operand producers ------------------------------------------------------
// SiLU with the approximate SFU ops (ex2.approx / rcp.approx, <= 2 ulp each): x / (1 + 2^(-x*log2 e))
__device__ __forceinline__ float silu_fast(float x) {
  float e, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * -1.4426950408889634f));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + e));
  return x * r;
}
// SiLU on 8 values with the five dependent stages issued stage-by-stage (8-way ILP)
__device__ __forceinline__ void silu_fast8(float v[8]) {
  float t[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) t[e] = v[e] * -1.4426950408889634f;
#pragma unroll
  for (int e = 0; e < 8; ++e) asm volatile("ex2.approx.ftz.f32 %0, %0;" : "+f"(t[e]));
#pragma unroll
  for (int e = 0; e < 8; ++e) t[e] += 1.0f;
#pragma unroll
  for (int e = 0; e < 8; ++e) asm volatile("rcp.approx.ftz.f32 %0, %0;" : "+f"(t[e]));
#pragma unroll
  for (int e = 0; e < 8; ++e) v[e] *= t[e];
}
// two fp32 -> fp16 hi pair + fp16 lo pair (lo = fp16(v - float(hi))).  Both conversions saturate to the largest
// finite fp16 (cvt .satfinite), so a value beyond the fp16 range degrades to a coarser finite value instead of
// inf - inf = NaN.
__device__ __forceinline__ void split2(float a, float b, uint32_t& hi, uint32_t& lo) {
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(b), "f"(a));
  const float2 hf = __half22float2(*reinterpret_cast<const __half2*>(&hi));
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(lo) : "f"(b - hf.y), "f"(a - hf.x));
}


// half mode: the hi parts of split2 only (same saturating rounding)
__device__ __forceinline__ uint32_t cvt_hi2(float a, float b) {
  uint32_t hi;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(b), "f"(a));
  return hi;
}

}  // namespace ptx
}  // namespace mcvd
