// tc_common.cuh -- inline-PTX helpers of the tensor-core convolution kernel (conv_tc.cu): mbarriers and bulk async
// copies.  sm_90a.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace fav {

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// Bounded wait: a protocol bug must surface as a trap (launch failure), never as a hung GPU.  The loop is written in
// PTX as one block: the same loop in C++ leaves the consumers a divergent path while wgmmas are in flight, and ptxas
// then serialises them (C7518).
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t.reg .b32 spin;\n\t.reg .b64 t0, now;\n\t"
      "mov.u32 spin, 0;\n\tmov.u64 t0, 0;\n"
      "LAB_WAIT:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra LAB_DONE;\n\t"
      "add.u32 spin, spin, 1;\n\t"
      "and.b32 spin, spin, 255;\n\t"
      "setp.ne.u32 p, spin, 0;\n\t"
      "@p bra LAB_WAIT;\n\t"
      "mov.u64 now, %%clock64;\n\t"
      "setp.eq.u64 p, t0, 0;\n\t"
      "@p mov.u64 t0, now;\n\t"
      "sub.s64 now, now, t0;\n\t"
      "setp.gt.s64 p, now, 4000000000;\n\t"  // ~2 s at 2 GHz
      "@p trap;\n\t"
      "bra LAB_WAIT;\n"
      "LAB_DONE:\n\t}" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
}  // namespace fav
