// conflux_b200/csrc/common.cuh -- shared device/host helpers (sm_90a only).
#pragma once
#include <cuda_runtime.h>

#include "../../include/conflux_b200.h"

#include <cstdint>
#include <cstdio>

namespace cflx {

// ---- error plumbing: every failure becomes a negative C-ABI code (cflx_status), never an exception ------------
void set_last_error(const char* fmt, ...);

#define CFLX_CUDA(call)                                                                                \
    do {                                                                                               \
        cudaError_t e__ = (call);                                                                      \
        if (e__ != cudaSuccess) {                                                                      \
            ::cflx::set_last_error("%s:%d: %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(e__)); \
            return CFLX_ERR_CUDA;                                                              \
        }                                                                                              \
    } while (0)

#define CFLX_TRY(call)              \
    do {                            \
        int rc__ = (call);          \
        if (rc__ != 0) return rc__; \
    } while (0)

static inline int64_t round_up(int64_t x, int64_t m) { return (x + m - 1) / m * m; }

// cudaFuncSetAttribute is per DEVICE: ranks may be threads of one process driving different GPUs, so the
// "already configured" bookkeeping is kept per device ordinal (values only grow; a benign race re-applies it).
struct PerDeviceMax {
    size_t v[64] = {0};
    // returns true when `want` exceeds what was configured on the current device (and records it)
    bool raise(size_t want) {
        int dev = 0;
        cudaGetDevice(&dev);
        dev &= 63;
        if (want > v[dev]) {
            v[dev] = want;
            return true;
        }
        return false;
    }
};

#ifdef __CUDACC__
// ---- mbarrier / bulk-copy (TMA engine, UBLKCP in SASS) PTX wrappers --------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
// non-blocking probe of a phase: true when the phase with this parity has completed
__device__ __forceinline__ bool mbar_test(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// 1-D bulk asynchronous copy global -> shared, completion counted in bytes on an mbarrier.
// dst/src 16-byte aligned, bytes a multiple of 16.
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

// FP64 tensor-core MMA (DMMA.8x8x4 in sm_90a SASS): D(8x8) += A(8x4, row) * B(4x8, col)
// lane l holds a = A[l>>2][l&3], b = B[l&3][l>>2], c0/c1 = C[l>>2][2*(l&3)+{0,1}]
__device__ __forceinline__ void dmma884(double& c0, double& c1, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                 : "+d"(c0), "+d"(c1)
                 : "d"(a), "d"(b));
}

// gpu-scope acquire/release accessors for the grid-wide pivot exchange
__device__ __forceinline__ int ld_acquire_gpu(const int* p) {
    int v;
    asm volatile("ld.acquire.gpu.global.b32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_gpu(int* p, int v) {
    asm volatile("st.release.gpu.global.b32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ double ld_cg_f64(const double* p) {
    double v;
    asm volatile("ld.global.cg.f64 %0, [%1];" : "=d"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ int ld_cg_s32(const int* p) {
    int v;
    asm volatile("ld.global.cg.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
#endif  // __CUDACC__

}  // namespace cflx
