// conflux_b200/csrc/gemm.cu -- FP64 tensor-core GEMM for the trailing-matrix update and the blocked TRSMs.
//
//   D[m][n] = beta * C[m][n] + alpha * sum_k AT[k][m] * B[k][n]          (all row-major, "TN" form)
//
// Replaces cblas_dgemm at /root/reference/src/conflux/lu/conflux_opt.hpp:1628-1632 (A11 -= A10Rcv * A01Rcv) and,
// through trsm.cu, the two cblas_dtrsm calls at :1347 and :1539.  Both operands are kept K-MAJOR in HBM
// (L is stored transposed, L^T[k][row]; U is U[k][col]) so that every operand row a CTA needs is one contiguous
// 1 KB segment: the producer warp stages tiles with 1-D bulk asynchronous copies (cp.async.bulk -> UBLKCP, the
// TMA engine) into a 4-stage shared-memory ring guarded by mbarriers, and 8 consumer warps run
// mma.sync.m8n8k4.f64 (DMMA.8x8x4 -- the native FP64 tensor instruction of sm_90a; wgmma has no f64 kind)
// on 64x32 warp tiles with accumulators in registers.  Shared-memory row stride is 132 doubles (== 4 mod 16) so
// both fragment loads (lane -> [k = lane&3][outer = lane>>2]) are bank-conflict free per half-warp.
#include <cstdlib>

#include "common.cuh"
#include "kernels.h"

namespace cflx {

namespace {
constexpr int BK = 16, STAGES = 4;

// WM x WN consumer warps, each owning a 64 x 32 tile of C: CTA tile (64*WM) x (32*WN).
//   <2,4,1>: 128x128, 8+1 warps, one CTA per SM (largest reuse per byte staged);
//   <1,4,2>:  64x128, 4+1 warps, TWO CTAs per SM so that one CTA's prologue/epilogue (operand fill, C read-modify-
//             write) overlaps the other's DMMA main loop.
template <int WM, int WN>
struct Cfg {
    static constexpr int BM = 64 * WM, BN = 32 * WN;
    static constexpr int LDA = BM + 4, LDB = BN + 4;  // strides == 4 (mod 16) doubles: conflict-free fragment loads
    static constexpr int NCONS = WM * WN, NTHREADS = (NCONS + 1) * 32;
    static constexpr size_t SMEM = (size_t)STAGES * BK * (LDA + LDB) * sizeof(double) + 2 * STAGES * sizeof(uint64_t);
};

// C may alias D (the trailing update is in place), so the read-only (.nc) path is off limits.  A plain coherent 16-byte
// load, written as non-volatile asm without a memory clobber: the compiler may schedule it freely among the stores of
// OTHER elements (each element is read exactly once, by the thread that later writes it; the data dependence keeps
// that load ahead of its own store), which preserves the batched-load memory-level parallelism.
__device__ __forceinline__ double2 ld_c2(const double* p) {
    double2 v;
    asm("ld.global.v2.f64 {%0, %1}, [%2];" : "=d"(v.x), "=d"(v.y) : "l"(p));
    return v;
}

template <int WM, int WN, int MINB>
__global__ void __launch_bounds__(Cfg<WM, WN>::NTHREADS, MINB) gemm_tn_kernel(GemmArgs g) {
    using C = Cfg<WM, WN>;
    constexpr int BM = C::BM, BN = C::BN, LDA = C::LDA, LDB = C::LDB, NCONS = C::NCONS;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    double* sA = reinterpret_cast<double*>(smem_raw);
    double* sB = sA + STAGES * BK * LDA;
    uint64_t* full = reinterpret_cast<uint64_t*>(sB + STAGES * BK * LDB);
    uint64_t* empty = full + STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
    const int KT = (g.K + BK - 1) / BK;

    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], NCONS);
        }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == NCONS) {
        // ===== producer: one bulk copy per operand row (lanes 0-15: A rows, 16-31: B rows) =====
        int wm = g.M - m0;
        wm = wm > BM ? BM : ((wm + 1) & ~1);
        int wn = g.N - n0;
        wn = wn > BN ? BN : ((wn + 1) & ~1);
        const int rr = lane & 15;
        for (int kt = 0; kt < KT; ++kt) {
            const int s = kt % STAGES, u = kt / STAGES;
            if (u > 0) mbar_wait(&empty[s], (u - 1) & 1);
            const int rows = min(BK, g.K - kt * BK);
            if (lane == 0) mbar_arrive_expect_tx(&full[s], (uint32_t)(rows * (wm + wn) * sizeof(double)));
            __syncwarp();
            if (rr < rows) {
                const int64_t k = (int64_t)kt * BK + rr;
                if (lane < 16)
                    bulk_g2s(sA + (s * BK + rr) * LDA, g.AT + k * g.ldat + m0, (uint32_t)(wm * sizeof(double)), &full[s]);
                else
                    bulk_g2s(sB + (s * BK + rr) * LDB, g.B + k * g.ldb + n0, (uint32_t)(wn * sizeof(double)), &full[s]);
            }
        }
        return;
    }

    // ===== consumers =====
    const int wm_off = (warp / WN) * 64, wn_off = (warp % WN) * 32;
    const int g4 = lane >> 2, t4 = lane & 3;
    double acc[8][4][2];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j][0] = acc[i][j][1] = 0.0;

    for (int kt = 0; kt < KT; ++kt) {
        const int s = kt % STAGES, u = kt / STAGES;
        mbar_wait(&full[s], u & 1);
        const double* a_s = sA + s * BK * LDA + wm_off + g4;
        const double* b_s = sB + s * BK * LDB + wn_off + g4;
        const int rows = min(BK, g.K - kt * BK);
#pragma unroll
        for (int kk = 0; kk < BK; kk += 4) {
            if (kk < rows) {
                double a[8], b[4];
#pragma unroll
                for (int i = 0; i < 8; ++i) a[i] = a_s[(kk + t4) * LDA + 8 * i];
#pragma unroll
                for (int j = 0; j < 4; ++j) b[j] = b_s[(kk + t4) * LDB + 8 * j];
#pragma unroll
                for (int i = 0; i < 8; ++i)
#pragma unroll
                    for (int j = 0; j < 4; ++j) dmma884(acc[i][j][0], acc[i][j][1], a[i], b[j]);
            }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[s]);
    }

    // ===== epilogue: registers <-> HBM directly, 16-byte accesses (each quad covers one 64 B row segment).
    // C and D may alias, so the compiler must not be left to order loads after earlier stores: all C loads of a
    // batch of two 8-row slabs are issued first (8 independent 16 B loads in flight per thread), then the stores.
    const double alpha = g.alpha, beta = g.beta;
    const bool use_c = (beta != 0.0);
#pragma unroll
    for (int ib = 0; ib < 8; ib += 2) {
        double2 cv[2][4];
#pragma unroll
        for (int ii = 0; ii < 2; ++ii) {
            const int row = m0 + wm_off + 8 * (ib + ii) + g4;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int col = n0 + wn_off + 8 * j + 2 * t4;
                cv[ii][j] = make_double2(0.0, 0.0);
                if (use_c && row < g.M && col < g.N)
                    cv[ii][j] = ld_c2(g.C + (int64_t)row * g.ldc + col);
            }
        }
#pragma unroll
        for (int ii = 0; ii < 2; ++ii) {
            const int row = m0 + wm_off + 8 * (ib + ii) + g4;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int col = n0 + wn_off + 8 * j + 2 * t4;
                if (row < g.M && col < g.N) {
                    double2 out;
                    out.x = fma(alpha, acc[ib + ii][j][0], beta * cv[ii][j].x);
                    out.y = fma(alpha, acc[ib + ii][j][1], beta * cv[ii][j].y);
                    *reinterpret_cast<double2*>(g.D + (int64_t)row * g.ldd + col) = out;
                }
            }
        }
    }
}
}  // namespace

namespace {
template <int WM, int WN, int MINB>
int setup_one() {
    static PerDeviceMax cfg;
    if (cfg.raise(Cfg<WM, WN>::SMEM))
        CFLX_CUDA(cudaFuncSetAttribute(gemm_tn_kernel<WM, WN, MINB>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)Cfg<WM, WN>::SMEM));
    return CFLX_OK;
}
template <int WM, int WN, int MINB>
int launch_one(const GemmArgs& g, cudaStream_t stream) {
    using C = Cfg<WM, WN>;
    CFLX_TRY((setup_one<WM, WN, MINB>()));
    dim3 grid((g.N + C::BN - 1) / C::BN, (g.M + C::BM - 1) / C::BM);
    gemm_tn_kernel<WM, WN, MINB><<<grid, C::NTHREADS, C::SMEM, stream>>>(g);
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}
int tile_variant() {  // default: 64x128 tile, two CTAs per SM;
                      // CFLX_GEMM_TILE=128 selects the 128x128 tile with one CTA per SM
    static int v = -1;
    if (v < 0) {
        const char* e = getenv("CFLX_GEMM_TILE");
        v = (e && atoi(e) == 128) ? 128 : 64;
    }
    return v;
}
}  // namespace

int gemm_tn_setup() {
    CFLX_TRY((setup_one<2, 4, 1>()));
    CFLX_TRY((setup_one<1, 4, 2>()));
    return CFLX_OK;
}

// Requirements: K % 4 == 0, N even, ldat/ldb/ldc/ldd even, all base pointers 16-byte aligned, ldat >= roundup2(M),
// ldb >= N.  M may be arbitrary (rows are masked).
int launch_gemm_tn(const GemmArgs& g, cudaStream_t stream) {
    if (g.M <= 0 || g.N <= 0 || g.K <= 0) return CFLX_OK;
    if ((g.K & 3) || (g.N & 1) || (g.ldat & 1) || (g.ldb & 1) || (g.ldc & 1) || (g.ldd & 1)) {
        set_last_error("gemm_tn: unsupported shape M=%d N=%d K=%d ld=(%lld,%lld,%lld,%lld)", g.M, g.N, g.K,
                       (long long)g.ldat, (long long)g.ldb, (long long)g.ldc, (long long)g.ldd);
        return CFLX_ERR_UNSUPPORTED;
    }
    if (tile_variant() == 64) return launch_one<1, 4, 2>(g, stream);
    return launch_one<2, 4, 1>(g, stream);
}

}  // namespace cflx
