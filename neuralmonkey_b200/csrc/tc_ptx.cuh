// PTX wrappers shared by the sm_90a kernels (gemm_tc.cu, decoder_step.cu): mbarrier, TMA,
// wgmma fences and shared-memory matrix descriptors.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace nm {

// ---------------------------------------------------------------------------
// PTX wrappers
// ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra WAIT_DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "WAIT_DONE:\n\t"
      "}" ::"r"(bar),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar,
                                            int32_t c0, int32_t c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
// expect `bytes` more transaction bytes on the barrier without arriving on it
__device__ __forceinline__ void mbar_expect_tx_only(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.expect_tx.relaxed.cta.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
constexpr float TC_LOG2E = 1.4426950408889634f;

// 2^x as ONE MUFU instruction.  exp2f() wraps the same MUFU.EX2 in a range fix for results below 2^-126
// (compare, halve, square: three more issue slots per element in epilogues that run once per logit); here such
// results flush to zero, which is what they contribute to a sum of probabilities anyway.
__device__ __forceinline__ float fast_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__device__ __forceinline__ uint32_t to_tf32(float x) {
  uint32_t u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
  return u;
}

// ---- wgmma (warpgroup MMA) ---------------------------------------------------------------------------
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accesses of accumulator registers across a wgmma wait
template <int R>
__device__ __forceinline__ void wgmma_fence_operands(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// Shared-memory matrix descriptor of a K-major operand tile in the 128-byte swizzle (rows of 128 bytes,
// 8-row atoms of 1 KB, tile base 1 KB aligned): start address >> 4 at [0,14), leading byte offset (unused
// by swizzled K-major layouts, 1) at [16,30), stride byte offset 1024 >> 4 at [32,46), layout 1 = 128B
// swizzle at [62,64).  Advancing `addr` by 32 bytes steps K by one instruction (8 tf32 / 16 fp16).
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t addr) {
  return (uint64_t)((addr & 0x3FFFFu) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) |
         ((uint64_t)1 << 62);
}

// The same for an MN-major 16-bit operand tile built from TMA boxes of 64 MN elements (128 B) x 64 k-rows in the
// 128-byte swizzle: 8-k-row atoms of 1 KB along K (stride byte offset 1024), the next 64 MN elements one 8 KB
// box further (leading byte offset 8192).  Advancing `addr` by 2048 bytes steps K by one instruction (16 rows).
__device__ __forceinline__ uint64_t gmma_desc_sw128_mn(uint32_t addr) {
  return (uint64_t)((addr & 0x3FFFFu) >> 4) | ((uint64_t)(8192 >> 4) << 16) | ((uint64_t)(1024 >> 4) << 32) |
         ((uint64_t)1 << 62);
}

// Stores into a K-major tile in the 128-byte swizzle (rows of 32 tf32 words), rounding to TF32 (cvt.rna): four
// words of 16-byte chunk `chunk`, or the single word `word`.
__device__ __forceinline__ void sw128_store4(uint8_t* tile, int row, int chunk, float4 v) {
  uint4 u = make_uint4(to_tf32(v.x), to_tf32(v.y), to_tf32(v.z), to_tf32(v.w));
  *reinterpret_cast<uint4*>(tile + row * 128 + ((chunk ^ (row & 7)) << 4)) = u;
}
__device__ __forceinline__ void sw128_store1(uint8_t* tile, int row, int word, float v) {
  *reinterpret_cast<uint32_t*>(tile + row * 128 + (((word >> 2) ^ (row & 7)) << 4) + ((word & 3) << 2)) = to_tf32(v);
}

}  // namespace nm
