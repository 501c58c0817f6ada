// Hopper asynchronous-copy and mbarrier primitives (sm_90a) shared by every kernel that stages data through shared
// memory: mbarrier set-up and waits, bulk copies (cp.async.bulk) and TMA tensor loads that complete on an mbarrier,
// bulk stores back to global memory, and the proxy fences between them.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace dz {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// Bytes from shared-memory address `base` up to the next 1024-byte boundary: `base + smem_pad_1024(base)` is the
// dynamic shared-memory base aligned for SWIZZLE_128B tiles (the launch adds 1024 bytes of slack).
__device__ __forceinline__ uint32_t smem_pad_1024(const void* base) {
  const uint32_t addr = smem_u32(base);
  return ((addr + 1023u) & ~1023u) - addr;
}

// ---- mbarriers ----------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
// Makes the initialised barriers visible to the async proxy (the bulk-copy / TMA units) before their first use.
__device__ __forceinline__ void fence_mbarrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// Arrive only where `pred` holds, without a branch: code between asynchronous warpgroup MMAs must stay free of
// divergent paths, or ptxas serialises the MMAs.
__device__ __forceinline__ void mbar_arrive_if(uint64_t* bar, bool pred) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %1, 0;\n@p mbarrier.arrive.shared::cta.b64 _, [%0];\n}\n" ::"r"(smem_u32(bar)),
               "r"((int)pred)
               : "memory");
}
// Arrive and add `bytes` to the phase's expected transaction count (the copies that complete on `bar`).
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}

// One lane of a converged warp.  With elect.sync ptxas knows that exactly one thread runs the guarded region and
// emits the bulk-copy / TMA instructions back to back instead of wrapping each in a loop over the possibly-active lanes.
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile("{\n .reg .pred P;\n elect.sync _|P, 0xffffffff;\n selp.u32 %0, 1, 0, P;\n}\n" : "=r"(pred));
  return pred != 0;
}

// ---- bulk copies and TMA ------------------------------------------------------------------------------------------
// global -> shared, `bytes` (multiple of 16) completing on `bar`
__device__ __forceinline__ void bulk_g2s(uint32_t dst_smem, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_smem),
               "l"(__cvta_generic_to_global(src)), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// shared -> global, tracked by the issuing thread's bulk groups
__device__ __forceinline__ void bulk_s2g(void* dst, const void* src_smem, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(__cvta_generic_to_global(dst)),
               "r"(smem_u32(src_smem)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// every committed store has completed
__device__ __forceinline__ void bulk_wait_group() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
// every committed store has finished reading its shared-memory source
__device__ __forceinline__ void bulk_wait_group_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }

__device__ __forceinline__ void tma_load_5d(uint32_t dst_smem, const void* map, uint64_t* bar, int c0, int c1, int c2, int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];" ::"r"(dst_smem),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}
__device__ __forceinline__ void prefetch_tensormap(const void* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}

// Orders this thread's generic-proxy shared-memory accesses before later async-proxy ones (a TMA refill of the slot, a
// bulk store of what the thread wrote).
__device__ __forceinline__ void fence_proxy_async_shared() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

}  // namespace dz
