// conflux_b200/csrc/wgmma.cuh -- what the wgmma trailing updates (ozaki.cu, tf32.cu) share: the TMA tensor loads, the
// wgmma group fences, the swizzled shared-memory descriptor of a K-major operand tile, and the host's tensor maps.
#pragma once
#include <cuda.h>

#include "common.cuh"

namespace cflx {

__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
            smem_u32(smem_dst)),
        "l"(map), "r"(c0), "r"(c1), "r"(smem_u32(bar))
        : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* map, int c0, int c1, int c2, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];" ::"r"(
            smem_u32(smem_dst)),
        "l"(map), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(bar))
        : "memory");
}
// shared-memory matrix descriptor of a K-major operand tile swizzled in SW-byte rows (SW = 64 or 128; 8-row groups 8 SW
// bytes apart): start address >> 4 | LBO (unused for swizzled K-major) = 1 at bit 16 | SBO = 8 SW >> 4 at bit 32 |
// the swizzle mode at bit 62 (SWIZZLE_64B 2, SWIZZLE_128B 1).  Stepping 32 bytes along K inside the swizzle atom adds 2
// to the start address field.
template <int SW>
__device__ __forceinline__ uint64_t smem_desc(uint32_t saddr) {
    static_assert(SW == 64 || SW == 128, "64- or 128-byte swizzle");
    return (uint64_t)((saddr & 0x3FFFF) >> 4) | (1ull << 16) | ((uint64_t)(8 * SW >> 4) << 32) |
           ((SW == 64 ? 2ull : 1ull) << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// ---------------------------------------------------------------------------------------------- host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
inline EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess && p) fn = (EncodeTiledFn)p;
        cudaGetLastError();
    }
    return fn;
}
// A tiled map of the rank-dimensional array at base (dims in elements, innermost first; strides in bytes of dimensions
// 1 ..), unit element strides, no interleave, 256-byte L2 promotion; what lies outside dims is read as zero
inline int make_tensor_map(CUtensorMap* map, CUtensorMapDataType type, cuuint32_t rank, const void* base,
                           const cuuint64_t* dims, const cuuint64_t* strides, const cuuint32_t* box,
                           CUtensorMapSwizzle swizzle) {
    EncodeTiledFn fn = encode_fn();
    if (!fn) {
        set_last_error("cuTensorMapEncodeTiled is not available from the driver");
        return CFLX_ERR_CUDA;
    }
    const cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    CUresult r = fn(map, type, rank, (void*)base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle,
                    CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_last_error("cuTensorMapEncodeTiled failed (%d) for %llu x %llu", (int)r, (unsigned long long)dims[0],
                       (unsigned long long)dims[1]);
        return CFLX_ERR_CUDA;
    }
    return CFLX_OK;
}

}  // namespace cflx
