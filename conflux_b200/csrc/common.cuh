// conflux_b200/csrc/common.cuh -- shared device/host helpers (sm_90a only).
#pragma once
#include <cuda_runtime.h>

#include "../../include/conflux_b200.h"

#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <initializer_list>
#include <mutex>
#include <type_traits>
#include <utility>

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

// A refused call of `who`: the error reads "<who>: refused, <what>"
inline int refuse(const char* who, const char* what, int status = CFLX_ERR_ARG) {
    set_last_error("%s: refused, %s", who, what);
    return status;
}
// CFLX_ERR_ARG naming the function and the condition that failed; REFUSE_FOR refuses in the name of a caller `who`
#define REFUSE_FOR(who, cond)                                 \
    do {                                                      \
        if (cond) return ::cflx::refuse((who), #cond);        \
    } while (0)
#define REFUSE_IF(cond) REFUSE_FOR(__func__, cond)

#define CFLX_TRY(call)              \
    do {                            \
        int rc__ = (call);          \
        if (rc__ != 0) return rc__; \
    } while (0)

static inline int64_t round_up(int64_t x, int64_t m) { return (x + m - 1) / m * m; }

// ---- owned device memory, pinned host memory, events and streams: released by their destructors, so a scope or an
// object that holds them frees them on every path.  Not copyable.  The current device must be the one they were made on.
//
// A device array of T, used as a T*.  alloc(n): max(n, 1) elements and a 4096-byte tail pad (bulk copies may
// over-read); alloc_exact(n): n elements, no pad.  grow(n) allocates again, with alloc, only when fewer than n elements are held.
template <class T = char>
struct DevBuf {
    T* p = nullptr;
    size_t n = 0;  // elements held
    DevBuf() = default;
    DevBuf(DevBuf&& o) noexcept : p(std::exchange(o.p, nullptr)), n(std::exchange(o.n, 0)) {}
    DevBuf& operator=(DevBuf&& o) noexcept {
        std::swap(p, o.p);
        std::swap(n, o.n);
        return *this;
    }
    ~DevBuf() { cudaFree(p); }
    void reset() {
        cudaFree(p);
        p = nullptr;
        n = 0;
    }
    int alloc(size_t count) { return alloc_bytes(count, std::max<size_t>(count, 1) * sizeof(T) + 4096); }
    int alloc_exact(size_t count) { return alloc_bytes(count, count * sizeof(T)); }
    bool holds(size_t count) const { return p && count <= n; }
    int grow(size_t count) { return holds(count) ? CFLX_OK : alloc(count); }
    operator T*() const { return p; }
    template <class U>
    U* as() const { return (U*)p; }

  private:
    int alloc_bytes(size_t count, size_t bytes) {
        reset();
        CFLX_CUDA(cudaMalloc((void**)&p, bytes));
        n = count;
        return CFLX_OK;
    }
};
// Buffers used together, grown together: unless every one holds n elements, all are freed, then all allocated, so the
// group is never held twice
template <class T>
int grow_together(std::initializer_list<DevBuf<T>*> group, size_t n) {
    if (std::all_of(group.begin(), group.end(), [n](const DevBuf<T>* b) { return b->holds(n); })) return CFLX_OK;
    for (DevBuf<T>* b : group) b->reset();
    for (DevBuf<T>* b : group) CFLX_TRY(b->alloc(n));
    return CFLX_OK;
}

// Page-locked host memory of n T, used as a T*
template <class T>
struct PinnedBuf {
    T* p = nullptr;
    PinnedBuf() = default;
    PinnedBuf(const PinnedBuf&) = delete;
    PinnedBuf& operator=(const PinnedBuf&) = delete;
    ~PinnedBuf() { cudaFreeHost(p); }
    int alloc(size_t n) {
        CFLX_CUDA(cudaMallocHost((void**)&p, n * sizeof(T)));
        return CFLX_OK;
    }
    operator T*() const { return p; }
};

// N events, made by create(flags); Events<1> (Event) is used as the cudaEvent_t itself
template <int N>
struct Events {
    cudaEvent_t e[N] = {};
    Events() = default;
    Events(Events&& o) noexcept { std::swap(e, o.e); }
    Events& operator=(Events&& o) noexcept {
        std::swap(e, o.e);
        return *this;
    }
    ~Events() {
        for (cudaEvent_t x : e)
            if (x) cudaEventDestroy(x);
    }
    int create(unsigned flags = cudaEventDefault) {
        for (cudaEvent_t& x : e) CFLX_CUDA(cudaEventCreateWithFlags(&x, flags));
        return CFLX_OK;
    }
    cudaEvent_t operator[](int i) const { return e[i]; }
    template <int M = N, class = std::enable_if_t<M == 1>>
    operator cudaEvent_t() const { return e[0]; }
};
using Event = Events<1>;

// A stream made by create(flags), or create(flags, priority)
struct Stream {
    cudaStream_t s = nullptr;
    Stream() = default;
    Stream(const Stream&) = delete;
    Stream& operator=(const Stream&) = delete;
    ~Stream() {
        if (s) cudaStreamDestroy(s);
    }
    int create(unsigned flags) {
        CFLX_CUDA(cudaStreamCreateWithFlags(&s, flags));
        return CFLX_OK;
    }
    int create(unsigned flags, int priority) {
        CFLX_CUDA(cudaStreamCreateWithPriority(&s, flags, priority));
        return CFLX_OK;
    }
    operator cudaStream_t() const { return s; }
};

// cudaFuncSetAttribute is per DEVICE: ranks may be threads of one process driving different GPUs, or several threads
// (ranks, or independent handles) driving the same one.  raise(want, set) runs set() on the current device when `want`
// exceeds what was configured there, and records it only once set() succeeded.  The lock makes every other thread
// that needs the attribute wait until it is in place: recording first and setting after would let a second thread
// launch with more shared memory than the function allows yet.
struct PerDeviceMax {
    std::mutex m;
    size_t v[64] = {0};
    template <class F>
    cudaError_t raise(size_t want, F&& set) {
        int dev = 0;
        cudaError_t e = cudaGetDevice(&dev);
        if (e != cudaSuccess) return e;
        dev &= 63;
        std::lock_guard<std::mutex> lk(m);
        if (want <= v[dev]) return cudaSuccess;
        e = set();
        if (e == cudaSuccess) v[dev] = want;
        return e;
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

// The Hopper f64 shapes, D(16x8) += A(16xk, row) * B(kx8, col), with g = lane>>2 and t = lane&3 (PTX ISA f64 fragment
// layouts).  Accumulators of all three: c0/c1 = C[g][2t+{0,1}], c2/c3 = C[g+8][2t+{0,1}].  Not volatile: the MMA has no
// side effect beyond its outputs, so ptxas may interleave the fragment loads of the next step with it.  gemm.cu issues
// m16n8k8 (its layout is checked against numpy by the GEMM tests); k4 and k16 run only in the rate probes of dbg.cu.
//   m16n8k4  (DMMA.16x8x4):  a0 = A[g][t], a1 = A[g+8][t];                                    b0 = B[t][g]
//   m16n8k8  (DMMA.16x8x8):  a0..a3 = A[g][t], A[g+8][t], A[g][t+4], A[g+8][t+4];           b0, b1 = B[t][g], B[t+4][g]
//   m16n8k16 (DMMA.16x8x16): a(2i), a(2i+1) = A[g][t+4i], A[g+8][t+4i] (i = 0..3);           b(i) = B[t+4i][g]
__device__ __forceinline__ void dmma16x8x4(double (&c)[4], const double (&a)[2], double b) {
    asm("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
        : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
        : "d"(a[0]), "d"(a[1]), "d"(b));
}
__device__ __forceinline__ void dmma16x8x8(double (&c)[4], const double (&a)[4], const double (&b)[2]) {
    asm("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
        : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b[0]), "d"(b[1]));
}
__device__ __forceinline__ void dmma16x8x16(double (&c)[4], const double (&a)[8], const double (&b)[4]) {
    asm("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, "
        "{%12,%13,%14,%15}, {%0,%1,%2,%3};"
        : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
        : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]),
          "d"(b[1]), "d"(b[2]), "d"(b[3]));
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
