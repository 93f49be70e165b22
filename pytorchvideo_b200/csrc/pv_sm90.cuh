// Thin inline-PTX wrappers for the Hopper (sm_90a) async machinery used by the implicit-GEMM kernels:
// mbarrier, TMA (cp.async.bulk.tensor), wgmma (fence / commit / wait, shared-memory descriptors).
#pragma once
#include <cuda.h>   // CUtensorMap (types only; the encode entry point is resolved at run time)
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "pv_wgmma.cuh"

namespace pv {
namespace sm90 {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

// ---- mbarrier -------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a pipeline bug must trap (-> CUDA error on the host) instead of hanging the GPU.  The whole loop is
// PTX (braces scope the labels), so the compiler sees neither a divergent loop nor a call: wgmma issued before the
// wait stays asynchronous across it.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      ".reg .u64 t0, t1;\n\t"
      "mov.u64 t0, %%clock64;\n\t"
      "WAIT:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%0], %1;\n\t"
      "@P bra DONE;\n\t"
      "mov.u64 t1, %%clock64;\n\t"
      "sub.u64 t1, t1, t0;\n\t"
      "setp.gt.u64 P, t1, 8000000000;\n\t"   // ~4 s at 2 GHz
      "@P trap;\n\t"
      "bra WAIT;\n\t"
      "DONE:\n\t"
      "}\n" ::"r"(bar), "r"(parity)
      : "memory");
}
// arrive only where `pred` is non-zero, without a branch around the instruction
__device__ __forceinline__ void mbar_arrive_if(uint32_t bar, bool pred) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %1, 0;\n\t"
      "@p mbarrier.arrive.shared::cta.b64 _, [%0];\n\t"
      "}\n" ::"r"(bar), "r"((uint32_t)pred)
      : "memory");
}

// ---- TMA ------------------------------------------------------------------------------------
// non-tensor bulk copy of `bytes` (a multiple of 16) from global to shared memory, completing on mbarrier `bar`
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}
__device__ __forceinline__ void prefetch_tmap(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const void* tmap, uint32_t bar, int c0,
                                            int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, "
      "{%3, %4}], [%2];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(tmap)), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const void* tmap, uint32_t bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(tmap)), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_5d(uint32_t dst, const void* tmap, uint32_t bar, int c0,
                                            int c1, int c2, int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, "
      "{%3, %4, %5, %6, %7}], [%2];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(tmap)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}

// ---- wgmma ----------------------------------------------------------------------------------
// Accumulators live in the registers of the issuing warpgroup.  fence: register / shared-memory writes of this
// thread are ordered before the next wgmma; commit closes a group of issued wgmma; wait<N> blocks until at most N
// groups are still in flight (their shared-memory operands may be overwritten only after that).
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator reads / writes across the asynchronous wgmma window
template <int R>
__device__ __forceinline__ void acc_fence(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// ---- descriptors ----------------------------------------------------------------------------
// K-major operand tile stored as rows of `swizzle_bytes` (128/64/32) bytes, 8-row swizzle atoms
// packed densely (SBO = 8 * swizzle_bytes).  Matches what TMA writes with the same swizzle mode.
// Field layout (PTX ISA, wgmma matrix descriptor): start>>4 [0,14), LBO>>4 [16,30), SBO>>4 [32,46),
// layout type [62,64): 1 = SW128, 2 = SW64, 3 = SW32.  Advancing K by 16 f16 (32 B) inside a swizzle row
// is +2 on the descriptor.
__host__ __device__ inline uint64_t make_kmajor_desc(uint32_t smem_addr, int swizzle_bytes) {
  const uint64_t layout = swizzle_bytes == 128 ? 1ull : (swizzle_bytes == 64 ? 2ull : 3ull);
  const uint64_t sbo = (uint64_t)(8 * swizzle_bytes) >> 4;
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);
  d |= (uint64_t)1 << 16;    // LBO (unused for swizzled K-major; canonical value 1)
  d |= sbo << 32;
  d |= layout << 62;
  return d;
}
// no-swizzle operand of 8-row x 16-byte core matrices: LBO = bytes between core matrices along K,
// SBO = bytes between 8-row groups along M / N
__host__ __device__ inline uint64_t make_noswz_desc(uint32_t smem_addr, uint32_t lbo, uint32_t sbo) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);
  d |= (uint64_t)(lbo >> 4) << 16;
  d |= (uint64_t)(sbo >> 4) << 32;
  return d;
}

}  // namespace sm90
}  // namespace pv
