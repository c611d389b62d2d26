// nvb_tma.cuh -- thin PTX wrappers for TMA bulk copies (cp.async.bulk, SASS UBLKCP) and the
// shared-memory mbarriers that track them. Hopper (sm_90a) instructions.
//
// A VoxelBlock is one contiguous, 16-byte-aligned run in the layer slab (4 KiB TSDF, 10 KiB
// ESDF), so a whole block moves HBM <-> shared memory with a single 1-D bulk copy issued by one
// thread; the other 255 threads of the CTA never touch an address register for it.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace nvb {
namespace tma {

__device__ __forceinline__ uint32_t smemAddr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbarInit(uint64_t* bar, uint32_t arrivals) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smemAddr(bar)), "r"(arrivals) : "memory");
}
// Make mbarrier.init (generic proxy) visible to the async proxy before the first bulk copy.
__device__ __forceinline__ void fenceBarrierInit() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// One arrival + the number of bytes the bulk copies of this phase will deliver.
__device__ __forceinline__ void mbarArriveExpectTx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smemAddr(bar)), "r"(bytes) : "memory");
}

// Plain arrival (completes a phase that expects no bytes).
__device__ __forceinline__ void mbarArrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smemAddr(bar)) : "memory");
}

__device__ __forceinline__ bool mbarTryWait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smemAddr(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbarWait(uint64_t* bar, uint32_t parity) {
  while (!mbarTryWait(bar, parity)) {
  }
}

// HBM -> shared memory, completion signalled on `bar` (complete_tx).
__device__ __forceinline__ void bulkLoad(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smemAddr(smem_dst)),
               "l"(gmem_src), "r"(bytes), "r"(smemAddr(bar))
               : "memory");
}

// Shared memory -> HBM, tracked by the issuing thread's bulk async-group.
__device__ __forceinline__ void bulkStore(void* gmem_dst, const void* smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gmem_dst), "r"(smemAddr(smem_src)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulkCommit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// Wait until all but the newest N committed groups have finished READING their shared-memory source.
template <int N>
__device__ __forceinline__ void bulkWaitRead() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
// Wait until all but the newest N committed groups are complete (writes performed).
template <int N>
__device__ __forceinline__ void bulkWait() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}
// Generic-proxy writes to shared memory -> visible to the async proxy (before a bulk store reads them).
__device__ __forceinline__ void fenceProxyAsyncShared() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

}  // namespace tma
}  // namespace nvb
