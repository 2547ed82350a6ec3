// conflux_b200/csrc/narrow.cuh -- the pieces of the narrow GEMM (solve.cu) that the residual kernels (refine.cu) share:
// the CTA shape, the arguments, and the double-buffered cp.async staging of B as k pairs.  See solve.cu for the design.
#pragma once
#include "common.cuh"

namespace cflx {
namespace {

constexpr int NW = 4;         // warps per CTA
constexpr int BM = 16 * NW;   // rows per CTA
constexpr int KC = 64;        // k rows per chunk (B in shared memory, A in registers)

struct NarrowArgs {
    int M, N, K;
    const double* A;
    int64_t lda;
    const double* B;
    int64_t ldb;
    const double* C;  // read only when beta != 0; may alias D
    int64_t ldc;
    double* D;
    int64_t ldd;
    double alpha, beta;
};

__device__ __forceinline__ void cp_async8(double* smem, const double* gmem, bool valid) {  // zero-fills when !valid
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;" ::"r"(smem_u32(smem)), "l"(gmem), "r"(valid ? 8 : 0)
                 : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

// k-pair rows of BN + 1 double2: the 8 lanes of a quarter warp (g = 0, 1; t = 0..3) read k pairs 2t + h, and
// 2t * (BN + 1) + g covers 8 distinct 16-byte bank groups
template <int NT>
struct NarrowCfg {
    static constexpr int BN = 8 * NT, LDP = BN + 1;
    static constexpr size_t STAGE = (size_t)KC / 2 * LDP;  // double2 per buffer
    static constexpr size_t SMEM = 2 * STAGE * sizeof(double2);
};

// B rows [kc, kc + KC) x columns [n0, n0 + BN) of chunk kc into one buffer, as k pairs
template <int NT>
__device__ __forceinline__ void stage_b(const NarrowArgs& g, int kc, int n0, double2* buf) {
    constexpr int BN = NarrowCfg<NT>::BN, LDP = NarrowCfg<NT>::LDP;
    double* d = reinterpret_cast<double*>(buf);
    for (int e = threadIdx.x; e < KC * BN; e += NW * 32) {
        const int kk = e / BN, n = e % BN, k = kc + kk, col = n0 + n;
        const bool ok = k < g.K && col < g.N;
        cp_async8(d + 2 * ((kk >> 1) * LDP + n) + (kk & 1), ok ? g.B + (int64_t)k * g.ldb + col : g.B, ok);
    }
    cp_async_commit();
}

}  // namespace
}  // namespace cflx
