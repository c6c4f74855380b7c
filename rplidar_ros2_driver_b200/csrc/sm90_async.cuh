// sm90_async.cuh -- PTX wrappers for the sm_90 asynchronous primitives of the scan kernels (scan_small.cu,
// scan_tma.cu): mbarriers, the 1-D bulk TMA copy, and the two-CTA cluster exchange through distributed shared memory.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace rpl {
namespace {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---- mbarrier ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(void* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_wait(void* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "LAB_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE;\n"
      "bra LAB_WAIT;\n"
      "DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
// producer-side wait: the ring is usually full, so let the hardware park the thread (suspend
// time hint, ns) instead of spinning through issue slots the consumer warps need
__device__ __forceinline__ void mbar_wait_relaxed(void* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "LAB_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1, %2;\n"
      "@p bra DONE;\n"
      "bra LAB_WAIT;\n"
      "DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity), "r"(20000u)
      : "memory");
}
__device__ __forceinline__ void mbar_arrive(void* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(void* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}

// 1-D bulk TMA copy global -> shared, completion counted in bytes on `bar`
__device__ __forceinline__ void tma_load_1d(void* dst, const void* src, uint32_t bytes, void* bar,
                                            uint64_t policy) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::
          "r"(smem_u32(dst)),
      "l"(src), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
      : "memory");
}

// ---- clusters ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
// all threads of both CTAs (exited threads would never arrive: call it with the whole block)
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release;\n\tbarrier.cluster.wait.acquire;" ::: "memory");
}
// shared::cluster address of `p`'s counterpart in CTA `rank` of the cluster
__device__ __forceinline__ uint32_t peer_addr(const void* p, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(smem_u32(p)), "r"(rank));
  return r;
}
// asynchronous store into a peer CTA's shared memory that counts its bytes on the peer's mbarrier `bar`:
// once the barrier's phase completes, the data is visible to the threads that waited on it
__device__ __forceinline__ void st_async_v4(uint32_t addr, uint4 v, uint32_t bar) {
  asm volatile("st.async.shared::cluster.mbarrier::complete_tx::bytes.v4.b32 [%0], {%1, %2, %3, %4}, [%5];" ::"r"(addr),
               "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w), "r"(bar)
               : "memory");
}
__device__ __forceinline__ void st_async_u32(uint32_t addr, uint32_t v, uint32_t bar) {
  asm volatile("st.async.shared::cluster.mbarrier::complete_tx::bytes.b32 [%0], %1, [%2];" ::"r"(addr), "r"(v),
               "r"(bar)
               : "memory");
}
// arrive on a barrier of the peer CTA, with the default semantics (release at CTA scope), as CUTLASS's cluster
// pipelines hand a buffer back to a peer CTA.  The caller must have consumed every value it read from the buffer the
// arrive hands back before a block barrier that precedes the arrive: nothing here orders those reads at cluster
// scope.  The .release.cluster form compiles to MEMBAR.ALL.GPU before the arrive, and every consumer warp of the
// cluster kernel waited behind that fence once per scan (DESIGN.md §5.1).
__device__ __forceinline__ void mbar_arrive_remote(uint32_t addr) {
  asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(addr) : "memory");
}
// plain load from the peer CTA's shared memory (ordered by a cluster barrier between the peer's store and it)
__device__ __forceinline__ uint32_t ld_peer_u32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared::cluster.u32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
  return v;
}
// wait for a phase completed by the peer's remote arrive: acquire at cluster scope, so that the peer's
// shared-memory accesses before its arrive are visible (or complete) here
__device__ __forceinline__ void mbar_wait_cluster(void* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "LAB_WAIT:\n"
      "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE;\n"
      "bra LAB_WAIT;\n"
      "DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}

}  // namespace
}  // namespace rpl
