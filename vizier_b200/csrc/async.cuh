// Asynchronous-copy primitives shared by the scoring kernels and the dataflow factorisation:
// cp.async (LDGSTS), mbarrier, TMA 2-D box loads and stores (cp.async.bulk.tensor), proxy fences, and the
// thread-block-cluster forms (cluster barrier, remote mbarrier arrive, TMA multicast).
#pragma once
#include <cuda.h>
#include <stdint.h>

namespace vzgp {

// ---- cp.async primitives ---------------------------------------------------------------
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc, bool valid) {
  const unsigned s = static_cast<unsigned>(__cvta_generic_to_shared(smem_dst));
  const int sz = valid ? 16 : 0;  // src-size 0 -> destination is zero-filled
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(s), "l"(gsrc), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory");
}
// ---- mbarrier / TMA (cp.async.bulk.tensor) primitives --------------------------------------
__device__ __forceinline__ unsigned smem_u32(const void* p) { return static_cast<unsigned>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, unsigned parity) {
  unsigned ok;
  do {
    asm volatile(
        "{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
  } while (!ok);
}
// 2-D tile load: box origin (c0 = column / innermost, c1 = row); completion bytes land on `bar`.
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];\n" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(smem_u32(bar))
      : "memory");
}
// 2-D tile store, the inverse of tma_load_2d: the box at smem_src (same layout and swizzle as a loaded box)
// goes to the box origin (c0, c1) of `map`.  Tracked by bulk async-groups, not by an mbarrier.
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, int c0, int c1, const void* smem_src) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%1, %2}], [%3];\n" ::"l"(
                   reinterpret_cast<uint64_t>(map)),
               "r"(c0), "r"(c1), "r"(smem_u32(smem_src))
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;\n" ::: "memory"); }
// At most N of this thread's bulk groups still read their shared-memory source (the source may be rewritten).
template <int N>
__device__ __forceinline__ void bulk_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;\n" ::"n"(N) : "memory");
}
// At most N of this thread's bulk groups are incomplete (their global writes are not yet performed).
template <int N>
__device__ __forceinline__ void bulk_wait() {
  asm volatile("cp.async.bulk.wait_group %0;\n" ::"n"(N) : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async;\n" ::: "memory"); }
// Generic-proxy shared-memory writes of this thread before later async-proxy (TMA store) reads of them.
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory"); }

// ---- thread-block clusters ---------------------------------------------------------------
__device__ __forceinline__ unsigned cluster_ctarank() {
  unsigned r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;\n" : "=r"(r));
  return r;
}
__device__ __forceinline__ unsigned cluster_nctarank() {
  unsigned r;
  asm volatile("mov.u32 %0, %%cluster_nctarank;\n" : "=r"(r));
  return r;
}
// Every thread of every CTA in the cluster: writes before it are visible cluster-wide after it.
__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release;\nbarrier.cluster.wait.acquire;\n" ::: "memory");
}
// Arrive on the mbarrier at the same shared-memory offset in CTA `rank` of the cluster (the own CTA
// included).  Used to release a ring stage whose next writer is a peer's TMA multicast.  This is the
// default (.release.cta) form, as CUTLASS's ClusterBarrier::arrive(cta_id) uses it: what must precede
// the peer's overwrite are this warp's shared-memory reads of the stage, and they have returned before
// the arrive issues, because the DMMAs that consume them come earlier in program order.  The
// .release.cluster form puts MEMBAR.ALL.CTA + MEMBAR.ALL.GPU before every arrive; in k_score it measured
// 5.14 ms against 4.49 ms for the C2 pool (H100 80GB HBM3, 400 W power limit).
__device__ __forceinline__ void mbar_arrive_cluster(const uint64_t* bar, unsigned rank) {
  asm volatile(
      "{\n.reg .b32 ra;\nmapa.shared::cluster.u32 ra, %0, %1;\nmbarrier.arrive.shared::cluster.b64 _, [ra];\n}\n" ::"r"(
          smem_u32(bar)),
      "r"(rank)
      : "memory");
}
// tma_load_2d into the same shared-memory offset of every CTA in `cta_mask`; each destination's
// mbarrier at the offset of `bar` receives the bytes.
__device__ __forceinline__ void tma_load_2d_multicast(void* smem_dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar,
                                                      uint16_t cta_mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%2, %3}], [%4], %5;\n" ::"r"(
          smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(smem_u32(bar)), "h"(cta_mask)
      : "memory");
}


}  // namespace vzgp
