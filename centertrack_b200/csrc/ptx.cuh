// Inline-PTX wrappers of the asynchronous-copy kernels (wgmma convolutions, heat-map decode): mbarriers, TMA and bulk
// copies, named barriers and the vector shared / non-coherent global accesses.
#pragma once
#include "common.cuh"
#include <cuda.h>

namespace ctb {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarriers ----
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
// makes the initialised barriers visible to the async proxy (TMA / bulk copies) and to the other threads
__device__ __forceinline__ void mbar_init_fence() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// arrive only where `pred` holds, without a branch (a branch between asynchronous MMAs makes ptxas serialise them)
__device__ __forceinline__ void mbar_arrive_if(uint32_t bar, bool pred) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %1, 0;\n\t@p mbarrier.arrive.shared::cta.b64 _, [%0];\n\t}"
               ::"r"(bar), "r"((uint32_t)pred) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}

// Watchdog report (ct_debug_watch): when set to host-mapped memory, a wait that never completes leaves
// (site, item, blockIdx.x, warp) in its 4 words before trapping, so a protocol bug can be located post mortem.
// The library is built without relocatable device code, so every translation unit that includes this header has its
// own copy of the pointer: set_mbar_watch() sets that unit's copy.
static __device__ volatile unsigned int* g_mbar_watch = nullptr;
static inline int set_mbar_watch(void* mapped_host_buf) {
  unsigned int* p = (unsigned int*)mapped_host_buf;
  return cudaMemcpyToSymbol(g_mbar_watch, &p, sizeof(p)) == cudaSuccess ? CT_OK : CT_ERR_CUDA;
}
// Waits for the phase with the given parity.  After 20 M unsuccessful polls the wait traps (a protocol bug must not
// hang the GPU); `site` and `item` only label the watchdog report.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity, int site = 0, int item = 0) {
  uint32_t done = 0, spins = 0;
  while (true) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.b32 %0, 1, 0, p;\n\t}"
        : "=r"(done) : "r"(bar), "r"(parity) : "memory");
    if (done) break;
    if (++spins > 20000000u) {
      volatile unsigned int* d = g_mbar_watch;
      if (d != nullptr && (threadIdx.x & 31) == 0) {
        d[0] = (unsigned)site; d[1] = (unsigned)item; d[2] = blockIdx.x; d[3] = threadIdx.x >> 5;
        __threadfence_system();
      }
      __trap();
    }
  }
}

// The same wait with its loop inside one asm block and no watchdog: for waits between asynchronous MMAs, where any
// branch the compiler sees makes ptxas serialise the MMAs.
__device__ __forceinline__ void mbar_wait_inline(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@!p bra WAIT_%=;\n\t}"
      ::"r"(bar), "r"(parity) : "memory");
}

// ---- async proxy: bulk and tensor (TMA) copies global -> shared, completing on an mbarrier ----
// generic-proxy shared-memory writes -> visible to the async proxy (tensor cores, TMA)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ void tma_3d(uint32_t dst, const CUtensorMap* map, int c0, int c1, int c2, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
      ::"r"(dst), "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(bar) : "memory");
}
__device__ __forceinline__ void tma_4d(uint32_t dst, const CUtensorMap* map, int c0, int c1, int c2, int c3, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];"
      ::"r"(dst), "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(bar) : "memory");
}

__device__ __forceinline__ void named_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
__device__ __forceinline__ void named_arrive(int id, int n) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(n) : "memory"); }

// ---- vector accesses ----
__device__ __forceinline__ uint4 lds16(uint32_t addr) {
  uint4 r;
  asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(addr));
  return r;
}
__device__ __forceinline__ void sts16(uint32_t addr, uint4 v) {
  asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ void sts32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ void sts_f2(uint32_t addr, float x, float y) {
  asm volatile("st.shared.v2.f32 [%0], {%1,%2};" ::"r"(addr), "f"(x), "f"(y) : "memory");
}
// M (a multiple of 4) consecutive floats from shared memory, 16 bytes per load
template <int M>
__device__ __forceinline__ void lds_f(uint32_t addr, float (&v)[M]) {
#pragma unroll
  for (int j4 = 0; j4 < M / 4; ++j4)
    asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(v[4 * j4]), "=f"(v[4 * j4 + 1]), "=f"(v[4 * j4 + 2]), "=f"(v[4 * j4 + 3])
                 : "r"(addr + 16u * j4));
}
__device__ __forceinline__ uint4 ldg_nc16(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ float4 ldg_nc_f4(const float* p) {
  float4 r;
  asm volatile("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
  return r;
}

}  // namespace ctb
