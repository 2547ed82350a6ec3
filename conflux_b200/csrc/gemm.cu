// conflux_b200/csrc/gemm.cu -- FP64 tensor-core GEMM for the trailing-matrix update and the blocked TRSMs.
//
//   D[m][n] = beta * C[m][n] + alpha * sum_k AT[k][m] * B[k][n]          (all row-major, "TN" form)
//
// Replaces cblas_dgemm at /root/reference/src/conflux/lu/conflux_opt.hpp:1628-1632 (A11 -= A10Rcv * A01Rcv) and,
// through trsm.cu, the two cblas_dtrsm calls at :1347 and :1539.  Both operands are kept K-MAJOR in HBM
// (L is stored transposed, L^T[k][row]; U is U[k][col]) so that every operand row a CTA needs is one contiguous
// 1 KB segment: the producer warp stages tiles with 1-D bulk asynchronous copies (cp.async.bulk -> UBLKCP, the
// TMA engine) into a 4-stage shared-memory ring guarded by mbarriers, and the consumer warps run
// mma.sync.m16n8k8.f64 (DMMA.16x8x8 in sm_90a SASS; wgmma has no f64 kind) on 64x32 warp tiles with accumulators in
// registers.  In a K tail of 4 rows (K % 8 == 4) the fragments of the 4 rows the copy did not fill are zeros, so no
// stale ring data reaches the MMA.  Shared-memory row strides are == 4 (mod 16) doubles so both fragment loads
// (lane -> [k = lane&3 (+4)][outer = lane>>2 (+8)]) are bank-conflict free per half-warp.
#include <cstdlib>

#include "common.cuh"
#include "kernels.h"

namespace cflx {

namespace {
constexpr int BK = 16, STAGES = 4;

// WM x WN consumer warps, each owning a 64 x 32 tile of C: CTA tile (64*WM) x (32*WN).
//   <2,4,1>: 128x128, 8+1 warps, one CTA per SM (largest reuse per byte staged; the default);
//   <1,4,2>:  64x128, 4+1 warps, TWO CTAs per SM so that one CTA's prologue/epilogue (operand fill, C read-modify-
//             write) overlaps the other's DMMA main loop.
// Register budget: ptxas sizes registers for the worst SM sub-partition, which holds 3 of the 9 (one CTA of <2,4,1>) or
// 10 (two CTAs of <1,4,2>) warps, so both run at 16384 / (3 * 32) -> 168 registers per thread.  The 64 accumulators
// take 128 of them, so a k-step holds all B fragments (8 doubles) but only one m16 tile's A fragment (4) at a time.
//
// C of the 128x128 tile goes through the ring (STAGE_C): as the last k-tiles drain the ring, the producer bulk-copies C
// into the freed stages, so the C reads of all but the last stage overlap the main loop and the epilogue reads shared
// memory instead of waiting on HBM slab after slab.  (An L2 prefetch of C at tile start measured slower: it competes
// with the operand stream and the concurrent pivot search for HBM and L2.)  A stage's A part (16 x LDA doubles) holds the 16-row slab
// of m16 tile i of warp row 0, its B part the same slab of warp row 1.  Row r of a slab starts at r * LDA + 4 (r & 1)
// doubles: even and odd rows are 64 bytes apart modulo 128, so the epilogue's 16-byte reads (a quarter-warp covers
// rows g, g + 1 at columns 2t..2t+1) are conflict-free, and the 16 rows end exactly at 16 * LDA.
template <int WM, int WN>
struct Cfg {
    static constexpr int BM = 64 * WM, BN = 32 * WN;
    static constexpr int LDA = BM + 4, LDB = BN + 4;  // strides == 4 (mod 16) doubles: conflict-free fragment loads
    static constexpr int NCONS = WM * WN, NTHREADS = (NCONS + 1) * 32;
    static constexpr bool STAGE_C = (WM == 2);
    static constexpr int NBAR = 2 * STAGES + (STAGE_C ? WM * STAGES : 0);  // full, empty (, one per C slab)
    static constexpr size_t SMEM = (size_t)STAGES * BK * (LDA + LDB) * sizeof(double) + NBAR * sizeof(uint64_t);
    static_assert(!STAGE_C || (LDA == LDB && 64 / 16 == STAGES), "one slab per warp row and stage, in both parts");
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
    uint64_t* cfull = empty + STAGES;  // STAGE_C: [warp row][i], the slab of m16 tile i has landed

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;

    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], NCONS);
        }
        if constexpr (C::STAGE_C)
            for (int b = 0; b < WM * STAGES; ++b) mbar_init(&cfull[b], 1);
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
        const int nkt = (g.K + BK - 1) / BK;
        const bool use_c = (g.beta != 0.0);
        for (int kt = 0; kt < nkt; ++kt) {
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
        if constexpr (C::STAGE_C) {
            // C slabs into the stages in the order they drain: (nkt + i) % STAGES was last used by k-tile nkt + i -
            // STAGES, or never (K < 64).  Lanes 0-15: the rows of warp row 0's slab, 16-31: warp row 1's.
            if (use_c)
                for (int i = 0; i < STAGES; ++i) {
                    const int s = (nkt + i) % STAGES, kt = nkt + i - STAGES;
                    if (kt >= 0) mbar_wait(&empty[s], (kt / STAGES) & 1);
                    const int wr = lane >> 4, r0 = m0 + 64 * wr + 16 * i;
                    const int rows = max(0, min(16, g.M - r0));
                    uint64_t* bar = &cfull[wr * STAGES + i];
                    if (rr == 0) mbar_arrive_expect_tx(bar, (uint32_t)(rows * wn * sizeof(double)));
                    __syncwarp();
                    if (rr < rows)
                        bulk_g2s(sA + (wr * STAGES + s) * BK * LDA + rr * LDA + 4 * (rr & 1),
                                 g.C + (int64_t)(r0 + rr) * g.ldc + n0, (uint32_t)(wn * sizeof(double)), bar);
                }
        }
        return;
    }

    // ===== consumers =====
    const int wm_off = (warp / WN) * 64, wn_off = (warp % WN) * 32;
    const int g4 = lane >> 2, t4 = lane & 3;
    // acc[i][j]: the m16n8 accumulator fragment of rows 16i.., columns 8j.. of the warp tile
    double acc[4][4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j][0] = acc[i][j][1] = acc[i][j][2] = acc[i][j][3] = 0.0;

    int kt = 0;  // after the loop: the number of k-tiles
    for (; kt * BK < g.K; ++kt) {
        const int s = kt % STAGES, u = kt / STAGES;
        mbar_wait(&full[s], u & 1);
        const double* a_s = sA + s * BK * LDA + wm_off + g4;
        const double* b_s = sB + s * BK * LDB + wn_off + g4;
        const int rows = min(BK, g.K - kt * BK);  // rows of this stage the copy filled, a multiple of 4
#pragma unroll
        for (int kk = 0; kk < BK; kk += 8) {
            if (kk < rows) {
                // K tail (rows == kk + 4): rows kk+4..kk+7 of the stage hold stale data, possibly NaN, which would
                // reach every output through the MMA; their fragments are zeros instead.
                const bool hi = kk + 4 < rows;
                const double* a_k = a_s + (kk + t4) * LDA;
                const double* b_k = b_s + (kk + t4) * LDB;
                // all B fragments of the k-step, the A fragments one m16 tile at a time (register budget, above)
                double b[4][2];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    b[j][0] = b_k[8 * j];
                    b[j][1] = hi ? b_k[4 * LDB + 8 * j] : 0.0;
                }
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const double a[4] = {a_k[16 * i], a_k[16 * i + 8], hi ? a_k[4 * LDA + 16 * i] : 0.0,
                                         hi ? a_k[4 * LDA + 16 * i + 8] : 0.0};
#pragma unroll
                    for (int j = 0; j < 4; ++j) dmma16x8x8(acc[i][j], a, b[j]);
                }
            }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[s]);
    }

    const double alpha = g.alpha, beta = g.beta;
    const bool use_c = (beta != 0.0);
    const int row0 = m0 + wm_off + g4, col0 = n0 + wn_off + 2 * t4;
    if constexpr (C::STAGE_C) {
        // ===== epilogue: C from the ring (see Cfg), slabs in the order the producer filled them; D straight to HBM
        // with 16-byte stores.  C and D may alias: every element's C is in shared memory before its store is issued.
        const int wr = warp / WN, nkt = kt;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const double* cs = sA + (wr * STAGES + (nkt + i) % STAGES) * BK * LDA + 4 * (g4 & 1) + wn_off + 2 * t4;
            if (use_c) mbar_wait(&cfull[wr * STAGES + i], 0);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int row = row0 + 16 * i + 8 * h;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const int col = col0 + 8 * j;
                    if (row < g.M && col < g.N) {
                        double2 cv = make_double2(0.0, 0.0);
                        if (use_c) cv = *reinterpret_cast<const double2*>(cs + (g4 + 8 * h) * LDA + 8 * j);
                        double2 out;
                        out.x = fma(alpha, acc[i][j][2 * h], beta * cv.x);
                        out.y = fma(alpha, acc[i][j][2 * h + 1], beta * cv.y);
                        *reinterpret_cast<double2*>(g.D + (int64_t)row * g.ldd + col) = out;
                    }
                }
            }
        }
    } else {
        // ===== epilogue: registers <-> HBM directly, 16-byte accesses (each quad covers one 64 B row segment).
        // C and D may alias, so the compiler must not be left to order loads after earlier stores: all C loads of an
        // 8-row slab are issued first (4 independent 16 B loads in flight per thread), then its stores.  One slab per
        // batch: with all 128 accumulator registers live, a second slab's loads would not fit the register budget.
#pragma unroll
        for (int sl = 0; sl < 8; ++sl) {
            const int row = row0 + 8 * sl;
            double2 cv[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int col = col0 + 8 * j;
                cv[j] = make_double2(0.0, 0.0);
                if (use_c && row < g.M && col < g.N) cv[j] = ld_c2(g.C + (int64_t)row * g.ldc + col);
            }
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int col = col0 + 8 * j;
                if (row < g.M && col < g.N) {
                    double2 out;
                    out.x = fma(alpha, acc[sl / 2][j][2 * (sl & 1)], beta * cv[j].x);
                    out.y = fma(alpha, acc[sl / 2][j][2 * (sl & 1) + 1], beta * cv[j].y);
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
    CFLX_CUDA(cfg.raise(Cfg<WM, WN>::SMEM, [&] {
        return cudaFuncSetAttribute(gemm_tn_kernel<WM, WN, MINB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg<WM, WN>::SMEM);
    }));
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
int tile_variant() {  // default: 128x128 tile, one CTA per SM (16 flop per operand byte at K = 256, against 10.7 for
                      // 64x128: measured faster on m16n8k8); CFLX_GEMM_TILE=64 selects the 64x128 tile, two CTAs per SM
    static int v = -1;
    if (v < 0) {
        const char* e = getenv("CFLX_GEMM_TILE");
        v = (e && atoi(e) == 64) ? 64 : 128;
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
