// Hopper (sm_90a) building blocks shared by the warpgroup-MMA kernels: shared-memory matrix descriptors, wgmma fences and
// groups, mbarriers and TMA tensor loads.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace iplan {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
// generic-proxy writes to shared memory -> visible to the async proxy (wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// Byte offset of 16-byte chunk `chunk` (0..7) of row `row` in a SWIZZLE_128B tile (rows of 128 B, base 1024-aligned)
__device__ __forceinline__ uint32_t swz128(int row, int chunk) {
    return (uint32_t)(row >> 3) * 1024u + (uint32_t)(row & 7) * 128u + (uint32_t)((chunk ^ (row & 7)) << 4);
}
// wgmma shared-memory matrix descriptor of a SWIZZLE_128B tile (rows of 128 B, base 1024-aligned, 8-row groups 1024 B apart:
// the stride byte offset).
//   K-major operand: a row holds 64 k of one m (or n); a k-block of 16 starts 32 B further; the leading byte offset is
//                    unused when K fits one swizzle atom.
//   MN-major operand (transposed wgmma): a row holds 64 consecutive m (or n) of one k, so 8 rows are 8 k and a k-block of
//                    16 starts 2048 B further; `lbo` is the distance between the 64-wide m (or n) blocks.
__device__ __forceinline__ uint64_t wgmma_desc(uint32_t smem_addr, uint32_t lbo = 16) {
    return (uint64_t)((smem_addr & 0x3FFFF) >> 4) | ((uint64_t)((lbo & 0x3FFFF) >> 4) << 16) | ((uint64_t)(1024 >> 4) << 32) |
           ((uint64_t)1 << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N_PENDING>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N_PENDING) : "memory"); }

// ---- mbarriers ------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
// make initialised barriers visible to the async proxy (TMA) before first use
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// wait until the phase of parity `parity` has completed (a fresh barrier counts its phase "before 0", parity 1, as complete)
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile("{\n\t.reg .pred done;\n"
                 "WAIT_%=:\n\t"
                 "mbarrier.try_wait.parity.shared::cta.b64 done, [%0], %1;\n\t"
                 "@!done bra WAIT_%=;\n\t}" ::"r"(bar), "r"(parity) : "memory");
}

// ---- TMA ------------------------------------------------------------------------------------------------------------------
// 3-D tiled tensor load into shared memory, completing `bar`'s transaction count by the box's bytes (out-of-bounds
// elements of the box are filled with zeros and counted too)
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const void* tmap, uint32_t bar, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
                 ::"r"(dst), "l"(tmap), "r"(bar), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const void* tmap) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(tmap) : "memory");
}

}  // namespace iplan
