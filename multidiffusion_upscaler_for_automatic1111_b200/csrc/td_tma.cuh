// TMA (cp.async.bulk.tensor) + mbarrier plumbing for sm_90a, raw PTX.
//
// Why TMA on this path: a CTA needs ~15 clipped sub-boxes of different tiles, and the
// per-warp chain "load -> wait -> add" of a register-staged kernel serialises DRAM
// latency.  A tiled tensor map takes signed box coordinates, clips against the tensor
// extent with zero fill, and keeps every box of the CTA in flight at once with no
// staging registers.  CONSTRAINT (CUDA 12.9): the innermost start
// coordinate must be 16-byte aligned (a misaligned c0 raises "illegal instruction"),
// so boxes are fetched as the aligned superset [floor(u0/VEC)*VEC, +BX+VEC) and the
// 2-byte-granular shift is applied when the threads read shared memory.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#ifdef __CUDACC__
namespace td {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
// make barrier inits / generic-proxy smem writes visible to the async (TMA) proxy
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t phase) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(phase)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t phase) {
    // bounded spin: a copy that never completes (bad descriptor) becomes a launch error, not a hung GPU
    for (uint32_t spins = 0; !mbar_try_wait(bar, phase); ++spins)
        if (spins > (1u << 26)) __trap();
}

// global -> shared, 3-D tiled box; completion is signalled on `bar` (complete_tx::bytes)
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* map, int c0, int c1, int c2, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(bar))
        : "memory");
}
// shared -> global, 3-D tiled box (out-of-bounds part of the box is not written)
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* map, int c0, int c1, int c2, const void* smem_src) {
    asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%1, %2, %3}], [%4];"
                 ::"l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(smem_src))
                 : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }

__device__ __forceinline__ uint4 lds128(const void* p) {
    uint4 v;
    asm volatile("ld.shared.v4.b32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(smem_u32(p)));
    return v;
}

}  // namespace td
#endif  // __CUDACC__

// ---- host side ---------------------------------------------------------------------------
// 3-D row-major tensor [planes][rows][cols] of `elem_size`-byte elements, box [1][box_rows][box_cols].
// Returns 0 on success; fills `out`.  Encoded through the driver entry point (no link-time libcuda).
int td_encode_tensor_map_3d(CUtensorMap* out, const void* base, int dtype, uint64_t planes, uint64_t rows, uint64_t cols,
                            uint32_t box_rows, uint32_t box_cols);
