// conflux_b200/csrc/chol.cu -- CONFCHOX: the reference's communication-avoiding Cholesky factorisation (A = L L^T, lower),
// re-designed for a grid of H100s.  BASELINE config C5: cholesky_miniapp --dim=32768 --tile=512 on 8 GPUs.
//
// Reference (relative to /root/reference/src/conflux/cholesky):
//   Cholesky.cpp:60-160        initialize(): grid / tile-size choice, buffers, input generation      -> cflx_chol_create,
//                                                                                                      cflx_chol_auto_grid/_tile
//   CholeskyIO.cpp:100-172     generateInputMatrixDistributed(): every v x v tile = lower(R^T R), srand(1),
//                              diagonal := 2 * Kappa * max row sum                                   -> cflx_chol_init_matrix_host
//   Cholesky.cpp:188-193       choleskyA00: LAPACKE_dpotrf on the diagonal tile                      -> potrf_tile_kernel
//   Cholesky.cpp:280-281,450   updateA10: cblas_dtrsm(Right, Lower, Trans, NonUnit) tile by tile     -> trsm_right_upper_T on L_kk^T
//   Cholesky.cpp:345-351,512+  computeA11: cblas_dgemm(N, T) tile by tile, k-slab of the z layer     -> gemm_tn on K-major panels
//   Cholesky.cpp:580-612       reduceA11: the next tile column is summed over the z layers            -> ncclReduce (k-communicator)
//   Cholesky.cpp:620-700       scatterA11 / A00 broadcast                                            -> ncclBroadcast of L_kk^T and of the
//                                                                                                      panel pieces
// GPU-first layout instead of the reference's tile objects (TileMatrix.h): every rank keeps its 2-D block-cyclic share
// of the matrix as ONE row-major Ml x Nl array in HBM (tile (gi, gj) on rank (gi % Px, gj % Py) at local tile (gi / Px,
// gj / Py); the lower triangle is meaningful), the tile column of a step is handled as a transposed (K-major) panel like
// in the LU path, so the TRSM and the rank-v update run on the same FP64 tensor-core GEMM (gemm.cu) on long contiguous
// operands instead of v x v tile calls.  The "A10 -> A01 representative" exchange of the reference (every rank needs the
// panel rows of its tile rows AND of its tile columns) is one grouped broadcast of the Px panel pieces to all ranks.
#include <climits>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <numeric>

#include "lu_state.h"

using namespace cflx;

// The grid's M is the padded order N, its Nt the reference's Kappa.  side: the panel pipeline of step k+1 (all NCCL
// traffic lives there) under the update of step k.  sv (cflx_chol_solve): inv(L_jj) blocks forward, inv(L_jj)^T
// backward; rows of real tiles.  eq: s is eq.*.r, scond eq.*.rowcnd.
struct cflx_chol : Handle {
    DevBuf<double> PT, LT, G /* [2] */, Bc /* [2] */, D, A00, W, Uinv, LinvT, acc;
    DevBuf<double> Q;  // scratch of the blocked tile Cholesky
    DevBuf<int> info;  // {-, first failing column, its min operand, -, the signed counts (LdltArgs::cnt)}
    int64_t ldp = 0, ldb = 0;
    // cflx_chol_factor_ldlt: the factor is signed (A = R S R^T), sgn holds S (M doubles, the same on every rank; made by
    // the first signed factorisation), tiny its pivot rule.  A plain factor has S = I.
    bool ldlt = false;
    double tiny = 0.0;
    DevBuf<double> sgn;
    Events<2> ev_col, ev_panel;
    SubComm j_comm;                  // grid row of one layer (color pi * Pz + pk, key pj), made by the first solve
    ~cflx_chol();  // the handle's device made current, the sub-communicators destroyed, then the members freed
};

namespace {

// ---------------------------------------------------------------------------------------------- diagonal tile
// The signed tile kernels' pivot rule (see potrf_tile_kernel): d, or copysign(tiny, d) (+tiny for +-0) when |d| < tiny;
// cnt (the one thread that counts, else null) += {replaced, positive, negative, zero}
__device__ __forceinline__ double ldlt_pivot(double d, double tiny, int* cnt) {
    const bool rep = fabs(d) < tiny;
    if (rep) d = d == 0.0 ? tiny : copysign(tiny, d);
    if (cnt) {
        cnt[0] += rep;
        cnt[1] += d > 0.0;
        cnt[2] += !(d > 0.0) && d != 0.0;
        cnt[3] += d == 0.0;
    }
    return d;
}
// the signs of a signed tile kernel's n columns and its counts out of shared memory (after its last __syncthreads)
__device__ __forceinline__ void ldlt_tile_out(const double* s_sg, const int* s_cnt, int n, const LdltArgs& sa) {
    __syncthreads();
    for (int e = threadIdx.x; e < n; e += blockDim.x) sa.sg[e] = s_sg[e];
    if (threadIdx.x < 4 && s_cnt[threadIdx.x]) atomicAdd(sa.cnt + threadIdx.x, s_cnt[threadIdx.x]);
}
// Cholesky of one v x v tile (row-major, lower triangle referenced) by ONE CTA: right-looking, 32-column blocks.
//   D   in: the tile; out: L in the lower triangle, zeros above
//   UT  out: L^T (upper triangular, row-major) -- the operand of the panel TRSM and what is broadcast
// info[0] = 1 + global index of the first non-positive pivot (0 = success), like LAPACK's dpotrf.  It is written with
// atomicCAS(info, 0, .), so the first failure of a factorisation is kept: after it, NaNs reach every later diagonal
// block, and each of those fails again.
constexpr int PB = 32;
//
// SIGNED (cflx_chol_factor_ldlt): the signed Cholesky A = R S R^T, S = diag(s), s_c = +-1, with R in D and S R^T (rows of
// R^T scaled by the signs) in UT and Uc.  Column c's pivot is d = a_cc - sum_{j<c} s_j r_cj^2; |d| < tiny becomes
// copysign(tiny, d) (+tiny for +-0), counted in sa.cnt[0]; then s_c = +1 for d > 0, else -1, r_cc = sqrt|d| and r_ic =
// (a_ic - sum_{j<c} r_ij s_j r_cj) / (s_c r_cc).  sa.sg receives the signs; sa.cnt[1..3] count the positive, negative
// and zero pivots; the failure *info records is an exactly zero d.  On s = +1 every operation is the unsigned one.
//
// D: v x v window (leading dimension ldd) of the tile, UT: the same window of L^T (leading dimension ldu); Uc (optional): a
// contiguous v x v copy of the factored block's L^T; col_off: global column of the window's first column (for *info)
template <bool SIGNED>
__global__ void __launch_bounds__(1024) potrf_tile_kernel(double* __restrict__ D, int v, int ldd, double* __restrict__ UT, int ldu,
                                                          double* __restrict__ Uc, int* __restrict__ info, int col_off,
                                                          LdltArgs sa) {
    extern __shared__ double sm[];
    double* Ld = sm;                 // [PB][PB + 1] factored diagonal block
    double* Xs = sm + PB * (PB + 1);  // [v][PB + 1] panel below it
    __shared__ int s_bad;
    __shared__ double s_sg[SIGNED ? 512 : 1];
    __shared__ int s_cnt[SIGNED ? 4 : 1];
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    if (t == 0) s_bad = 0;
    if (SIGNED && t < 4) s_cnt[t] = 0;
    for (int jb = 0; jb < v; jb += PB) {
        const int nb = min(PB, v - jb), m = v - jb - nb;
        for (int e = t; e < nb * nb; e += blockDim.x) Ld[(e / nb) * (PB + 1) + e % nb] = D[(size_t)(jb + e / nb) * ldd + jb + e % nb];
        __syncthreads();
        if (warp == 0) {  // lane = row of the block, the row lives in registers
            double a[PB];
#pragma unroll
            for (int c = 0; c < PB; ++c) a[c] = (lane < nb && c <= lane && c < nb) ? Ld[lane * (PB + 1) + c] : 0.0;
#pragma unroll
            for (int c = 0; c < PB; ++c) {
                if (c < nb) {
                    double d = __shfl_sync(0xffffffffu, a[c], c), sgc = 1.0;
                    if (SIGNED) {
                        d = ldlt_pivot(d, sa.tiny, lane == 0 ? s_cnt : nullptr);
                        sgc = d > 0.0 ? 1.0 : -1.0;
                        if (lane == 0) s_sg[jb + c] = sgc;
                        if (d == 0.0 && lane == 0 && s_bad == 0) s_bad = col_off + jb + c + 1;
                    } else if (!(d > 0.0) && lane == 0 && s_bad == 0) {
                        s_bad = col_off + jb + c + 1;
                    }
                    const double sq = SIGNED ? sqrt(fabs(d)) : sqrt(d);
                    if (lane == c) a[c] = sq;
                    else if (lane > c) a[c] = a[c] / (SIGNED ? sgc * sq : sq);
#pragma unroll
                    for (int c2 = c + 1; c2 < PB; ++c2) {
                        double l2 = __shfl_sync(0xffffffffu, a[c], c2);  // L[c2][c]
                        if (SIGNED) l2 *= sgc;
                        if (lane >= c2) a[c2] = fma(-a[c], l2, a[c2]);
                    }
                }
            }
#pragma unroll
            for (int c = 0; c < PB; ++c)
                if (lane < nb && c < nb) Ld[lane * (PB + 1) + c] = (c <= lane) ? a[c] : 0.0;
        }
        __syncthreads();
        // the factored block goes back (zeros above its diagonal) and into UT transposed
        for (int e = t; e < nb * nb; e += blockDim.x) {
            const int r = e / nb, c = e % nb;
            const double x = Ld[r * (PB + 1) + c];
            D[(size_t)(jb + r) * ldd + jb + c] = x;
            UT[(size_t)(jb + c) * ldu + jb + r] = SIGNED && c <= r ? s_sg[jb + c] * x : x;  // UT[c][r] = s_c L[r][c] (zero for c > r)
        }
        // panel below: X = P * L_d^-T, one thread per row (forward substitution against the block in shared memory)
        for (int i = t; i < m; i += blockDim.x) {
            double* prow = D + (size_t)(jb + nb + i) * ldd + jb;
            double x[PB];
#pragma unroll
            for (int c = 0; c < PB; ++c) x[c] = c < nb ? prow[c] : 0.0;
#pragma unroll
            for (int c = 0; c < PB; ++c) {
                if (c < nb) {
                    double s = x[c];
#pragma unroll
                    for (int q = 0; q < c; ++q) s = fma(-x[q], SIGNED ? s_sg[jb + q] * Ld[c * (PB + 1) + q] : Ld[c * (PB + 1) + q], s);
                    x[c] = s / (SIGNED ? s_sg[jb + c] * Ld[c * (PB + 1) + c] : Ld[c * (PB + 1) + c]);
                }
            }
#pragma unroll
            for (int c = 0; c < PB; ++c) {
                if (c < nb) {
                    prow[c] = x[c];
                    Xs[i * (PB + 1) + c] = x[c];
                    UT[(size_t)(jb + c) * ldu + jb + nb + i] = SIGNED ? s_sg[jb + c] * x[c] : x[c];   // L^T (S R^T)
                }
            }
        }
        __syncthreads();
        // trailing block (lower triangle, row i >= column j): T[i][j] -= X[i][:] . X[j][:]
        const int tiles = (m + 31) / 32;
        for (int tt = warp; tt < tiles * tiles; tt += (blockDim.x >> 5)) {
            const int ti = tt / tiles, tj = tt % tiles;
            if (tj > ti) continue;
            const int j = tj * 32 + lane;
            // 8 rows per iteration: the 8 loads of T are issued together (they are L2 round trips of a single SM), then
            // the dot products against the shared-memory panel, then the 8 stores
#pragma unroll 1
            for (int i0 = 0; i0 < 32; i0 += 8) {
                double tv[8];
#pragma unroll
                for (int q = 0; q < 8; ++q) {
                    const int i = ti * 32 + i0 + q;
                    tv[q] = (i < m && j < m && j <= i) ? D[(size_t)(jb + nb + i) * ldd + jb + nb + j] : 0.0;
                }
#pragma unroll
                for (int q = 0; q < 8; ++q) {
                    const int i = ti * 32 + i0 + q;
                    if (i < m && j < m && j <= i) {
                        double s = 0.0;
#pragma unroll
                        for (int c = 0; c < PB; ++c)
                            s = fma(Xs[i * (PB + 1) + c], SIGNED ? s_sg[jb + c] * Xs[j * (PB + 1) + c] : Xs[j * (PB + 1) + c], s);
                        tv[q] -= s;
                    }
                }
#pragma unroll
                for (int q = 0; q < 8; ++q) {
                    const int i = ti * 32 + i0 + q;
                    if (i < m && j < m && j <= i) D[(size_t)(jb + nb + i) * ldd + jb + nb + j] = tv[q];
                }
            }
        }
        __syncthreads();
    }
    // zeros above the diagonal of D / below the diagonal of UT
    for (int e = t; e < v * v; e += blockDim.x) {
        const int r = e / v, c = e % v;
        if (c > r) {
            D[(size_t)r * ldd + c] = 0.0;
            UT[(size_t)c * ldu + r] = 0.0;
        }
    }
    if (Uc != nullptr) {
        __syncthreads();
        for (int e = t; e < v * v; e += blockDim.x) Uc[e] = UT[(size_t)(e / v) * ldu + e % v];
    }
    if (SIGNED) ldlt_tile_out(s_sg, s_cnt, v, sa);
    if (t == 0 && s_bad) atomicCAS(info, 0, s_bad);
}

// Cholesky of ONE 128 x 128 diagonal block held entirely in shared memory (the building block of potrf_tile): all 512
// threads take part in every phase -- 32-column diagonal blocks on warp 0 (row per lane), the rows below
// by forward substitution (one row per thread), the trailing part one element per thread from shared memory.  D / UT are
// windows of the tile (leading dimensions ldd / ldu), Uc a contiguous copy of L^T for the block-column solve.
constexpr int QBK = 128;
constexpr int QPITCH = QBK + 1;
constexpr int QTHREADS = 512;
// SIGNED: the signed Cholesky of the block, as potrf_tile_kernel's.
template <bool SIGNED>
__global__ void __launch_bounds__(QTHREADS) potrf128_kernel(double* __restrict__ D, int ldd, double* __restrict__ UT, int ldu,
                                                        double* __restrict__ Uc, int* __restrict__ info, int col_off,
                                                        LdltArgs sa) {
    extern __shared__ double As[];  // [QBK][QPITCH], lower triangle
    __shared__ int s_bad;
    __shared__ double s_sg[SIGNED ? QBK : 1];
    __shared__ int s_cnt[SIGNED ? 4 : 1];
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    if (t == 0) s_bad = 0;
    if (SIGNED && t < 4) s_cnt[t] = 0;
    for (int e = t; e < QBK * QBK; e += QTHREADS) {
        const int r = e / QBK, c = e % QBK;
        As[r * QPITCH + c] = (c <= r) ? D[(size_t)r * ldd + c] : 0.0;
    }
    __syncthreads();
    for (int jb = 0; jb < QBK; jb += PB) {
        const int m = QBK - jb - PB;
        if (warp == 0) {  // 32 x 32 diagonal block in place, lane = row (shared memory: a register array of 32 doubles that is
                          // indexed by the unrolled column loop ends up in local memory, which is what made the old kernel slow)
            double* B = As + jb * QPITCH + jb;
            for (int c = 0; c < PB; ++c) {
                double d = B[c * QPITCH + c], sgc = 1.0;
                if (SIGNED) {
                    d = ldlt_pivot(d, sa.tiny, lane == 0 ? s_cnt : nullptr);
                    sgc = d > 0.0 ? 1.0 : -1.0;
                    if (lane == 0) s_sg[jb + c] = sgc;
                    if (d == 0.0 && lane == 0 && s_bad == 0) s_bad = col_off + jb + c + 1;
                } else if (!(d > 0.0) && lane == 0 && s_bad == 0) {
                    s_bad = col_off + jb + c + 1;
                }
                const double sq = SIGNED ? sqrt(fabs(d)) : sqrt(d);
                double l = 0.0;
                if (lane == c) B[c * QPITCH + c] = sq;
                else if (lane > c) {
                    l = B[lane * QPITCH + c] / (SIGNED ? sgc * sq : sq);
                    B[lane * QPITCH + c] = l;
                }
                __syncwarp();
#pragma unroll 4
                for (int c2 = c + 1; c2 < PB; ++c2) {
                    const double l2 = SIGNED ? sgc * B[c2 * QPITCH + c] : B[c2 * QPITCH + c];  // (s_c) L[c2][c], broadcast
                    if (lane >= c2) B[lane * QPITCH + c2] = fma(-l, l2, B[lane * QPITCH + c2]);
                }
                __syncwarp();
            }
        }
        __syncthreads();
        if (m <= 0) break;
        // rows below: X = P * L_d^-T, one row per thread, in place in shared memory (L_d is a broadcast read)
        if (t < m) {
            double* prow = As + (jb + PB + t) * QPITCH + jb;
            const double* Ld = As + jb * QPITCH + jb;
#pragma unroll 4
            for (int c = 0; c < PB; ++c) {
                double sacc = prow[c];
                for (int q = 0; q < c; ++q) sacc = fma(-prow[q], SIGNED ? s_sg[jb + q] * Ld[c * QPITCH + q] : Ld[c * QPITCH + q], sacc);
                prow[c] = sacc / (SIGNED ? s_sg[jb + c] * Ld[c * QPITCH + c] : Ld[c * QPITCH + c]);
            }
        }
        __syncthreads();
        // trailing part (lower triangle): T[i][k] -= X[i][:] . X[k][:], one element per thread and pass (signed: the
        // block's signs held in registers)
        double sgr[SIGNED ? PB : 1];
        if (SIGNED)
#pragma unroll
            for (int c = 0; c < PB; ++c) sgr[c] = s_sg[jb + c];
        for (int e = t; e < m * m; e += QTHREADS) {
            const int i = e / m, k = e % m;
            if (k > i) continue;
            const double* xi = As + (jb + PB + i) * QPITCH + jb;
            const double* xk = As + (jb + PB + k) * QPITCH + jb;
            double sacc = 0.0;
#pragma unroll
            for (int c = 0; c < PB; ++c) sacc = fma(xi[c], SIGNED ? sgr[c] * xk[c] : xk[c], sacc);
            As[(jb + PB + i) * QPITCH + jb + PB + k] -= sacc;
        }
        __syncthreads();
    }
    // L into the tile (zeros above its diagonal), L^T into UT and into the contiguous copy
    for (int e = t; e < QBK * QBK; e += QTHREADS) {
        const int r = e / QBK, c = e % QBK;
        D[(size_t)r * ldd + c] = As[r * QPITCH + c];            // (zeros above the diagonal were loaded as zeros)
        const double lt = SIGNED && c >= r ? s_sg[r] * As[c * QPITCH + r] : As[c * QPITCH + r];  // (s_r) L^T[r][c] = L[c][r]
        UT[(size_t)r * ldu + c] = lt;
        Uc[e] = lt;
    }
    if (SIGNED) ldlt_tile_out(s_sg, s_cnt, QBK, sa);
    if (t == 0 && s_bad) atomicCAS(info, 0, s_bad);
}

// out[r][x] = sg[r] X[r][x] for x < n (both leading dimension ld): a row r per blockIdx.y
__global__ void row_signs_kernel(const double* __restrict__ X, int64_t ld, int n, const double* __restrict__ sg,
                                 double* __restrict__ out) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, r = blockIdx.y;
    if (x < n) out[(int64_t)r * ld + x] = sg[r] * X[(int64_t)r * ld + x];
}
// zeros above the diagonal of D (= L) and below the diagonal of UT (= L^T)
__global__ void tri_clean_kernel(double* __restrict__ D, double* __restrict__ UT, int v) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= v * v) return;
    const int r = e / v, c = e % v;
    if (c > r) {
        D[e] = 0.0;
        UT[(size_t)c * v + r] = 0.0;
    }
}

// D[r][c] = PT[c][r] (diagonal tile out of the transposed panel) / A11 tile <- D
__global__ void tile_from_panel_kernel(const double* __restrict__ PT, int64_t ldp, int v, double* __restrict__ D) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e < v * v) D[e] = PT[(int64_t)(e % v) * ldp + e / v];
}
__global__ void tile_store_kernel(const double* __restrict__ D, int v, double* __restrict__ A, int64_t lda) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e < v * v) A[(int64_t)(e / v) * lda + e % v] = D[e];
}
// Bc[c][t * v + x] = G_piece(j % Px)[c][(j / Px) * v - row1(j % Px) + x] for the local column tiles t (global j = (lj0 + t) * Py + pj)
struct GatherArgs {
    const double* G;       // Px pieces, piece p = [v][ld_p] with ld_p = its active rows rounded up to even
    int64_t piece_stride;
    double* Bc;
    int64_t ldb;
    int v, Px, Py, pj, lj0, ntiles, gfirst, Ml;
    const double* sg;      // the v signs of the step (signed update), or null
};
// SIGNED: Bc's row c times a.sg[c], the sign of contraction index c (S_k R_jk^T of the signed update)
template <bool SIGNED>
__global__ void gather_cols_kernel(GatherArgs a) {
    const int t = blockIdx.x, c = blockIdx.y;
    const int j = (a.lj0 + t) * a.Py + a.pj;            // global tile index of this local column tile
    const int p = j % a.Px;
    const int d = a.gfirst - p;
    const int first = d <= 0 ? 0 : (d + a.Px - 1) / a.Px;   // first local tile row of piece p that holds a tile >= gfirst
    const int rows = a.Ml - first * a.v;
    const int64_t ldg = max(2, (rows + 1) & ~1);
    const double* src = a.G + (int64_t)p * a.piece_stride + (int64_t)c * ldg + (int64_t)(j / a.Px - first) * a.v;
    double* dst = a.Bc + (int64_t)c * a.ldb + (int64_t)t * a.v;
    if (SIGNED) {
        const double sg = a.sg[c];
        for (int x = threadIdx.x; x < a.v; x += blockDim.x) dst[x] = sg * src[x];
    } else {
        for (int x = threadIdx.x; x < a.v; x += blockDim.x) dst[x] = src[x];
    }
}
// sum of squares of the lower triangle of the real tiles (global row >= global column, global row < Nt v: the column
// is then below that bound too) of a local block-cyclic array: partials[blockIdx.x] = this CTA's share;
// launch_sum_partials then adds them in index order, so every call rounds the same way
__global__ void sumsq_lower_kernel(const double* __restrict__ X, Layout L, double* __restrict__ partials) {
    double s = 0.0;
    const int64_t total = (int64_t)L.Ml * L.Nl, nreal = (int64_t)L.Nt * L.v;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        const int lr = (int)(e / L.Nl), lc = (int)(e % L.Nl);
        const int64_t gr = L.row<int64_t>(lr);
        if (gr < nreal && gr >= L.col<int64_t>(lc)) s = fma(X[e], X[e], s);
    }
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    __shared__ double w[32];
    if ((threadIdx.x & 31) == 0) w[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x < 32) {
        s = threadIdx.x < (blockDim.x >> 5) ? w[threadIdx.x] : 0.0;
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (threadIdx.x == 0) partials[blockIdx.x] = s;
    }
}
// info[2] = info[1], or INT_MAX when this rank saw no failure: the operand of the ncclMin that finds the first failing
// column over the grid
__global__ void info_min_operand_kernel(int* info) { info[2] = info[1] ? info[1] : INT_MAX; }
// validation: transposed panel of column block t out of the stored factor, the diagonal tile masked to its lower triangle
__global__ void extract_l_panel_T_kernel(const double* __restrict__ A, int64_t lda, int row0, int col0, int n, Layout L,
                                         int t, double* __restrict__ PT, int64_t ldp) {
    const int v = L.v;
    __shared__ double tile[32][33];
    const int r0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    for (int dy = threadIdx.y; dy < 32; dy += blockDim.y) {
        const int r = r0 + dy, c = c0 + threadIdx.x;
        double x = 0.0;
        if (r < n && c < v) {
            const int lr = row0 + r;
            const int64_t gr = L.row<int64_t>(lr), gc = (int64_t)t * v + c;
            x = gr >= gc ? A[(int64_t)lr * lda + col0 + c] : 0.0;
        }
        tile[dy][threadIdx.x] = x;
    }
    __syncthreads();
    for (int dy = threadIdx.y; dy < 32; dy += blockDim.y) {
        const int c = c0 + dy, r = r0 + threadIdx.x;
        if (r < n && c < v) PT[(int64_t)c * ldp + r] = tile[threadIdx.x][dy];
    }
}

int chol_pick_nb(int v) {
    for (int nb : {128, 64, 32, 16, 8, 4})
        if (v % nb == 0) return nb;
    return 0;
}

// Broadcast the Px pieces of the (transposed) panel of column block t to every rank and apply
//   X[i][j] -= L[i][t] * L[j][t]^T   to the local tiles with global tile row i >= tile column j >= jmin (lower triangle),
// each z layer with its own slab of the v contraction indices.  piece_rows0(p) = first local row of piece p.
int piece_ld(const cflx_chol* ch, int gfirst, int p) { return chol_piece_ld(*ch, gfirst, p); }
// Broadcast the Px pieces of the (transposed) panel of column block t (rows of global tiles >= gfirst) to every rank into
// buffer set `buf`, and assemble the column operand for the local column tiles with global index >= jmin.
// carry_signs (the signed factorisation): the diagonal owner's piece also carries the step's v signs, written after
// its v ld_p values (the owner put them there), and every rank copies them into its sign vector.  The gather applies the
// signs whenever the factor is signed.
int broadcast_pieces(cflx_chol* ch, int t, int gfirst, int jmin, int buf, cudaStream_t s, bool carry_signs = false) {
    const int v = ch->v, Px = ch->Px, Py = ch->Py, Pz = ch->Pz, Ml = ch->Ml, Nl = ch->Nl;
    const int pjt = t % Py;
    const int64_t piece_stride = (int64_t)v * ch->ldp;
    double* G = ch->G + (int64_t)buf * Px * piece_stride;
    double* Bc = ch->Bc + (int64_t)buf * v * ch->ldb;
    if (ch->P > 1) {
        const int pd = t % Px;
        CFLX_NCCL(ncclGroupStart());
        for (int p = 0; p < Px; ++p) {
            const int rows = Ml - first_local_tile(gfirst, p, Px) * v;
            const bool signs = carry_signs && p == pd;
            if (rows <= 0 && !signs) continue;
            const int root = (p * Py + pjt) * Pz;
            double* dst = G + (int64_t)p * piece_stride;
            const double* src = (ch->rank == root) ? ch->LT : dst;
            CFLX_NCCL(ncclBroadcast(src, dst, (size_t)v * (piece_ld(ch, gfirst, p) + signs), ncclDouble, root,
                                    ch->comm->world, s));
        }
        CFLX_NCCL(ncclGroupEnd());
        if (carry_signs)
            CFLX_CUDA(cudaMemcpyAsync(ch->sgn + (int64_t)t * v, G + (int64_t)pd * piece_stride + (int64_t)v * piece_ld(ch, gfirst, pd),
                                      (size_t)v * sizeof(double), cudaMemcpyDeviceToDevice, s));
    } else {
        CFLX_CUDA(cudaMemcpyAsync(G, ch->LT, (size_t)v * piece_ld(ch, gfirst, 0) * sizeof(double), cudaMemcpyDeviceToDevice, s));
    }
    const int lj0 = first_local_tile(jmin, ch->pj, Py);
    const int ntc = Nl / v - lj0;
    if (ntc <= 0) return CFLX_OK;
    CFLX_TRY(launch_gather_cols(G, piece_stride, Bc, ch->ldb, v, Px, Py, ch->pj, lj0, ntc, gfirst, Ml, s,
                                ch->ldlt ? ch->sgn + (int64_t)t * v : nullptr));
    ch->launches++;
    return CFLX_OK;
}
// X[i][j] -= L[i][t] * L[j][t]^T on the local tiles with global tile row i >= tile column j, j in the local column tiles
// [lj_lo, lj_hi) (global index >= jmin; lower triangle), each z layer with its own slab of the v contraction indices.
// SMs the persistent int8 update leaves to the look-ahead panel pipeline on the side stream (CFLX_CHOL_LEAVE)
static int chol_leave_sms() {
    static int leave = -1;
    if (leave < 0) {
        const char* e = getenv("CFLX_CHOL_LEAVE");
        leave = e ? atoi(e) : 8;
        if (leave < 0) leave = 0;
        if (leave > 100) leave = 100;
    }
    return leave;
}

// fp64: the FP64 kernel whatever the handle's update (the validation's update); otherwise the handle's update on the
// operands split_planes split from buffer set buf
int update_columns(cflx_chol* ch, int gfirst, int jmin, int buf, double* X, int lj_lo, int lj_hi, cudaStream_t s,
                   bool fp64 = false) {
    const int v = ch->v, Px = ch->Px, Py = ch->Py, Ml = ch->Ml, Nl = ch->Nl;
    const int pi = ch->pi, pj = ch->pj, pk = ch->pk;
    const int64_t piece_stride = (int64_t)v * ch->ldp;
    const double* G = ch->G + (int64_t)buf * Px * piece_stride;
    const double* Bc = ch->Bc + (int64_t)buf * v * ch->ldb;
    const int lj0 = first_local_tile(jmin, pj, Py);              // Bc column 0 corresponds to this local tile
    const int my_first = first_local_tile(gfirst, pi, Px);        // first local tile row of MY piece
    const int64_t ldg = piece_ld(ch, gfirst, pi);
    // One launch per GROUP of local tile columns: wide enough (>= ~8192 rows x columns of v) to fill the machine; the rows
    // start at the diagonal of the group's first column, so later columns of a group also update a few tiles above their
    // own diagonal (upper triangle: never read) -- a few per cent of extra flops instead of many half-empty launches.
    const int lj_end = std::min(lj_hi, Nl / v);
    const int my_rows = Ml - my_first * v;                          // rows of my piece = rows of the A planes
    for (int lj = std::max(lj_lo, lj0); lj < lj_end;) {
        const int j = lj * Py + pj;                               // global tile column of the group's first column
        const int li = first_local_tile(j, pi, Px);               // first local tile row with global index >= j
        const int M = Ml - li * v;
        if (M <= 0) break;                                        // later columns have even fewer rows
        int gcols = std::max(1, (8192 + M - 1) / M);
        gcols = std::min(gcols, lj_end - lj);
        GemmArgs g{};
        g.M = M; g.N = gcols * v; g.K = ch->nlayr;
        g.AT = G + (int64_t)pi * piece_stride + (int64_t)pk * ch->nlayr * ldg + (int64_t)(li - my_first) * v;
        g.ldat = ldg;
        g.B = Bc + (int64_t)pk * ch->nlayr * ch->ldb + (int64_t)(lj - lj0) * v;
        g.ldb = ch->ldb;
        g.C = X + (int64_t)li * v * Nl + (int64_t)lj * v;
        g.ldc = Nl;
        g.D = const_cast<double*>(g.C);
        g.ldd = Nl;
        g.alpha = -1.0; g.beta = 1.0;
        if (fp64) CFLX_TRY(launch_gemm_tn(g, s));
        else CFLX_TRY(ch->update.apply(g, (li - my_first) * v, (lj - lj0) * v, chol_leave_sms(), s));
        ch->launches++;
        lj += gcols;
    }
    (void)my_rows;
    return CFLX_OK;
}
// the operands of one update sweep, split for a split kind: my piece (rows) and the gathered column operand, this
// layer's slab
int split_planes(cflx_chol* ch, int gfirst, int jmin, int buf, cudaStream_t s) {
    if (!ch->update.splits()) return CFLX_OK;
    const int v = ch->v, Px = ch->Px;
    const int64_t piece_stride = (int64_t)v * ch->ldp;
    const double* G = ch->G + (int64_t)buf * Px * piece_stride;
    const double* Bc = ch->Bc + (int64_t)buf * v * ch->ldb;
    const int my_first = first_local_tile(gfirst, ch->pi, Px);
    const int rows = ch->Ml - my_first * v;
    const int ncols = ch->Nl - first_local_tile(jmin, ch->pj, ch->Py) * v;
    const int64_t ldg = piece_ld(ch, gfirst, ch->pi);
    const double* A = G + (int64_t)ch->pi * piece_stride + (int64_t)ch->pk * ch->nlayr * ldg;
    const double* B = Bc + (int64_t)ch->pk * ch->nlayr * ch->ldb;
    if (rows > 0) CFLX_TRY(ch->update.split_a(A, ldg, rows, s));
    if (ncols > 0) CFLX_TRY(ch->update.split_b(B, ch->ldb, 0, ncols, s));
    ch->launches += 2;
    return CFLX_OK;
}
int broadcast_and_update(cflx_chol* ch, int t, int jmin, bool below_only, double* X, cudaStream_t s) {
    const int gfirst = below_only ? t + 1 : t;
    CFLX_TRY(broadcast_pieces(ch, t, gfirst, jmin, 0, s));
    return update_columns(ch, gfirst, jmin, 0, X, 0, ch->Nl / ch->v, s, true);
}

size_t potrf_tile_smem(int v) { return ((size_t)PB * (PB + 1) + (size_t)v * (PB + 1)) * sizeof(double); }
}  // namespace

namespace cflx {
size_t potrf_tile_scratch(int v) { return (v % QBK == 0 && v >= 2 * QBK) ? (size_t)3 * QBK * QBK + (size_t)2 * QBK * v : 0; }

// raise-only: a smaller v (another object, a test hook) never lowers the limit a live object relies on
int potrf_setup(int v) {
    static PerDeviceMax tile_cfg, blk_cfg;
    CFLX_CUDA(tile_cfg.raise(potrf_tile_smem(v), [&] {
        cudaError_t e = cudaFuncSetAttribute(potrf_tile_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)potrf_tile_smem(v));
        if (e == cudaSuccess)
            e = cudaFuncSetAttribute(potrf_tile_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)potrf_tile_smem(v));
        return e;
    }));
    CFLX_CUDA(blk_cfg.raise(QBK * QPITCH * sizeof(double), [&] {
        cudaError_t e = cudaFuncSetAttribute(potrf128_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(QBK * QPITCH * sizeof(double)));
        if (e == cudaSuccess)
            e = cudaFuncSetAttribute(potrf128_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(QBK * QPITCH * sizeof(double)));
        return e;
    }));
    return CFLX_OK;
}

int potrf_block128(double* D, int ldd, double* UT, int ldu, double* Uc, int* info, int col0, cudaStream_t s,
                   const LdltArgs* sa) {
    if (sa)
        potrf128_kernel<true><<<1, QTHREADS, QBK * QPITCH * sizeof(double), s>>>(D, ldd, UT, ldu, Uc, info, col0, *sa);
    else
        potrf128_kernel<false><<<1, QTHREADS, QBK * QPITCH * sizeof(double), s>>>(D, ldd, UT, ldu, Uc, info, col0, LdltArgs{});
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}

// Cholesky of the v x v diagonal tile.  One CTA alone is far too slow for a 512 x 512 tile (it would sit on
// the critical path of every step), so the tile is itself factored in 128-wide block columns: the 128 x 128 diagonal block on one CTA, the
// block column below it by ONE GEMM with the inverted block, the trailing part of the tile by one rank-128 GEMM -- both on
// the whole GPU (FP64 DMMA kernel).  Tiles that are not a multiple of 128 (tests), or Q == nullptr, keep the one-CTA kernel.
// With sa, the signed Cholesky (potrf_tile_kernel): block jb's signs go to sa->sg + jb, and the rank-128 update of the
// trailing part is T -= X S X^T, its second operand (and A00's copy of the block column) S X^T.
int potrf_tile(double* D, double* A00, double* Q, int* info, int col0, int v, cudaStream_t s, int64_t* launches,
               const LdltArgs* sa) {
    constexpr int QB = 128;
    if (v % QB != 0 || v < 2 * QB || Q == nullptr) {
        if (sa) potrf_tile_kernel<true><<<1, 1024, potrf_tile_smem(v), s>>>(D, v, v, A00, v, nullptr, info, col0, *sa);
        else potrf_tile_kernel<false><<<1, 1024, potrf_tile_smem(v), s>>>(D, v, v, A00, v, nullptr, info, col0, LdltArgs{});
        CFLX_CUDA(cudaGetLastError());
        return CFLX_OK;
    }
    double* U128 = Q;                          // [QB][QB]  L_d^T of the current diagonal block, contiguous
    double* Ui = U128 + QB * QB;               // [QB][QB]  its inverse
    double* Li = Ui + QB * QB;                 // [QB][QB]  (unit-lower companion of launch_diag_inverses, unused)
    double* XT0 = Li + QB * QB;                // [QB][v]   block column below the diagonal block, transposed
    double* XT = XT0 + (size_t)QB * v;         // [QB][v]   ... after the solve
    static_assert(QB == QBK, "block width of the tile Cholesky");
    for (int jb = 0; jb < v; jb += QB) {
        const int m = v - jb - QB;
        LdltArgs sb{};
        if (sa) sb = LdltArgs{sa->tiny, sa->sg + jb, sa->cnt};
        CFLX_TRY(potrf_block128(D + (size_t)jb * v + jb, v, A00 + (size_t)jb * v + jb, v, U128, info, col0 + jb, s,
                                sa ? &sb : nullptr));
        ++*launches;
        if (m <= 0) break;
        const int64_t ldx = m;
        CFLX_TRY(launch_extract_panel_T(D, v, jb + QB, jb, m, QB, XT0, ldx, s));
        CFLX_TRY(launch_diag_inverses(U128, QB, QB, Ui, Li, s));
        CFLX_TRY(trsm_right_upper_T(U128, Ui, QB, QB, XT0, XT, ldx, m, s));          // X^T = L_d^-1 P^T (signed: S R_d^T)
        CFLX_TRY(launch_store_panel_T(D, v, jb + QB, jb, m, QB, XT, ldx, s));
        const double* XS = XT;                                                        // S X^T (X^T unsigned)
        if (sa) {
            row_signs_kernel<<<dim3((m + 255) / 256, QB), 256, 0, s>>>(XT, ldx, m, sb.sg, XT0);
            CFLX_CUDA(cudaGetLastError());
            ++*launches;
            XS = XT0;
        }
        CFLX_CUDA(cudaMemcpy2DAsync(A00 + (size_t)jb * v + jb + QB, (size_t)v * sizeof(double), XS, ldx * sizeof(double),
                                    (size_t)m * sizeof(double), QB, cudaMemcpyDeviceToDevice, s));
        GemmArgs g{};                                                                 // T -= X X^T (X S X^T)
        g.M = m; g.N = m; g.K = QB;
        g.AT = XT; g.ldat = ldx;
        g.B = XS; g.ldb = ldx;
        g.C = D + (size_t)(jb + QB) * v + jb + QB; g.ldc = v;
        g.D = D + (size_t)(jb + QB) * v + jb + QB; g.ldd = v;
        g.alpha = -1.0; g.beta = 1.0;
        CFLX_TRY(launch_gemm_tn(g, s));
        *launches += 6;
    }
    tri_clean_kernel<<<(v * v + 255) / 256, 256, 0, s>>>(D, A00, v);
    CFLX_CUDA(cudaGetLastError());
    ++*launches;
    return CFLX_OK;
}

int launch_gather_cols(const double* G, int64_t piece_stride, double* Bc, int64_t ldb, int v, int Px, int Py, int pj,
                       int lj0, int ntiles, int gfirst, int Ml, cudaStream_t s, const double* sg) {
    GatherArgs ga{G, piece_stride, Bc, ldb, v, Px, Py, pj, lj0, ntiles, gfirst, Ml, sg};
    if (sg) gather_cols_kernel<true><<<dim3(ntiles, v), 128, 0, s>>>(ga);
    else gather_cols_kernel<false><<<dim3(ntiles, v), 128, 0, s>>>(ga);
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}

int launch_sumsq_lower(const double* X, const Layout& L, double* partials, double* out, cudaStream_t s) {
    sumsq_lower_kernel<<<SUMSQ_PARTIALS, 256, 0, s>>>(X, L, partials);
    CFLX_CUDA(cudaGetLastError());
    return launch_sum_partials(partials, SUMSQ_PARTIALS, out, s);
}

int launch_extract_l_panel_T(const double* A, int64_t lda, int row0, int col0, int n, const Layout& L, int t, double* PT,
                             int64_t ldp, cudaStream_t s) {
    if (n <= 0) return CFLX_OK;
    dim3 grid((n + 31) / 32, (L.v + 31) / 32), block(32, 8);
    extract_l_panel_T_kernel<<<grid, block, 0, s>>>(A, lda, row0, col0, n, L, t, PT, ldp);
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}
}  // namespace cflx

namespace {
// Panel pipeline of step k on stream s: z-reduce of tile column k, Cholesky of the diagonal tile, L_kk^T down the grid
// column, the panel solve, the stores, and (k < Nt - 1) the broadcast of the panel pieces into buffer set k & 1.
int panel_step(cflx_chol* ch, int k, cudaStream_t s) {
    const int v = ch->v, Px = ch->Px, Py = ch->Py, Pz = ch->Pz, Ml = ch->Ml, Nl = ch->Nl;
    const int pi = ch->pi, pj = ch->pj, pk = ch->pk;
    const int pik = k % Px, pjk = k % Py;
    const int loff = (k / Py) * v;
    const int row0 = first_local_tile(k, pi, Px) * v;        // my first row at or below tile k
    const int row1 = first_local_tile(k + 1, pi, Px) * v;    // ... strictly below tile k
    const int n0 = Ml - row0, n1 = Ml - row1;
    const int64_t ld = std::max<int64_t>(2, round_up(n0, 2));    // panel from the diagonal tile down
    const int64_t ld1 = piece_ld(ch, k + 1, pi);                 // rows strictly below tile k (what is broadcast)
    const bool on_col = (pj == pjk);
    const bool owner = on_col && pi == pik && pk == 0;
    // (4 of the previous step) tile column k summed over the z layers                  Cholesky.cpp:580-612
    if (on_col && n0 > 0) {
        CFLX_TRY(launch_extract_panel_T(ch->A11, Nl, row0, loff, n0, v, ch->PT, ld, s));
        ch->launches++;
        if (Pz > 1) CFLX_NCCL(ncclReduce(ch->PT, ch->PT, (size_t)v * ld, ncclDouble, ncclSum, 0, ch->k_comm.c, s));
    }
    // (1) Cholesky of the diagonal tile                                                 Cholesky.cpp:188-193
    if (owner) {
        tile_from_panel_kernel<<<(v * v + 255) / 256, 256, 0, s>>>(ch->PT, ld, v, ch->D);
        const LdltArgs sa{ch->tiny, ch->sgn + (int64_t)k * v, ch->info + 4};
        CFLX_TRY(potrf_tile(ch->D, ch->A00, ch->Q, ch->info + 1, k * v, v, s, &ch->launches, ch->ldlt ? &sa : nullptr));
        tile_store_kernel<<<(v * v + 255) / 256, 256, 0, s>>>(ch->D, v, ch->A11 + (int64_t)row0 * Nl + loff, Nl);
        CFLX_CUDA(cudaGetLastError());
        ch->launches += 3;
    }
    if (k == ch->Nt - 1) return CFLX_OK;
    // L_kk^T to the ranks that hold the tile column (layer 0)                           Cholesky.cpp:680-690
    if (on_col && pk == 0 && Px > 1)
        CFLX_NCCL(ncclBroadcast(ch->A00, ch->A00, (size_t)v * v, ncclDouble, pik, ch->i_comm.c, s));
    // (2) tile column: A10 <- A10 * L_kk^-T                                              Cholesky.cpp:280-281,450-451
    if (on_col && pk == 0 && n1 > 0) {
        CFLX_TRY(launch_diag_inverses(ch->A00, v, ch->nb, ch->Uinv, ch->LinvT, s));
        // PT rows are relative to row0 (ld); the solve works on the window below the diagonal tile and the result is
        // repacked with the leading dimension of the broadcast piece (ld1)
        CFLX_TRY(trsm_right_upper_T(ch->A00, ch->Uinv, v, ch->nb, ch->PT + (row1 - row0), ch->W, ld, n1, s));
        CFLX_CUDA(cudaMemcpy2DAsync(ch->LT, ld1 * sizeof(double), ch->W, ld * sizeof(double), (size_t)n1 * sizeof(double), v,
                                    cudaMemcpyDeviceToDevice, s));
        CFLX_TRY(launch_store_panel_T(ch->A11, Nl, row1, loff, n1, v, ch->LT, ld1, s));
        ch->launches += 2 * (v / ch->nb) + 1;
    }
    // the signs of step k ride on the owner's piece (after its v ld1 values)
    if (owner && ch->ldlt && ch->P > 1)
        CFLX_CUDA(cudaMemcpyAsync(ch->LT + (int64_t)v * ld1, ch->sgn + (int64_t)k * v, (size_t)v * sizeof(double),
                                  cudaMemcpyDeviceToDevice, s));
    // the reference's A10 -> A01 representative exchange                                 Cholesky.cpp:205-330
    return broadcast_pieces(ch, k, k + 1, k + 1, k & 1, s, ch->ldlt);
}

// ---------------------------------------------------------------------------------------------- solve, A X = B
// After the factorisation, layer 0's A11 holds L: tile (gi, gj), gi >= gj, on rank (gi % Px, gj % Py, 0) at local tile
// (gi / Px, gj / Py), the diagonal tiles with zeros above the diagonal.  The solve reads nothing else: not the tiles above
// the diagonal (leftovers of the update), not the local tiles with a global index >= Nt, not the layers pk != 0.  It
// is the engine's row-partial sweep L Y = B (W seeded with B's rows on the ranks (pi, 0, 0); Y_t kept at the owner's
// local column t / Py of Z), then its column-partial sweep L^T X = Y.  The grid row and column are those of layer 0
// (j_comm / i_comm, one layer each); the layers pk != 0 only join the final all-reduce.
SolveFactor chol_solve_factor(cflx_chol* ch) {
    return SolveFactor{*ch, ch->A11, first_local_tile(ch->Nt, ch->pi, ch->Px) * ch->v, &ch->j_comm, &ch->i_comm, 1,
                       ch->ldlt ? ch->sgn.p : nullptr};
}

// First call after a factorisation: the grid-row communicator (once per object), the inverses of the nb x nb diagonal
// blocks of every owned diagonal tile, and on the ranks that seed W, the row of B of each of their real local rows.
int chol_solve_prepare(cflx_chol* ch) {
    cflx_comm* c = ch->comm;
    if (c->world_size > 1 && !ch->j_comm.c) CFLX_TRY(make_sub(c, ch->pi * ch->Pz + ch->pk, ch->pj, ch->Py, &ch->j_comm));
    if (ch->pk == 0) {
        const SolveFactor f = chol_solve_factor(ch);
        CFLX_TRY(solve_inverses(&ch->sv, f, true));
        if (ch->pj == 0 && !ch->sv.rows) {  // local row r of a real tile holds global row ch->row(r)
            std::vector<int> rows(std::max(f.rows, 1), 0);
            for (int r = 0; r < f.rows; ++r) rows[r] = ch->row(r);
            CFLX_TRY(solve_set_rows(&ch->sv.rows, rows, c->stream));
        }
    }
    ch->sv.ready = true;
    return CFLX_OK;
}

// One solve with the factor of the last successful factorisation (cflx_chol_solve, cflx_chol_solve_local); B host or
// device, X may be null (the solution then stays in ch->sv.X).
int chol_sweeps(cflx_chol* ch, int nrhs, const double* B, int ldb, double* X, int ldx) {
    if (!ch->sv.ready) CFLX_TRY(chol_solve_prepare(ch));
    const SolveFactor f = chol_solve_factor(ch);
    SolveCache* sc = &ch->sv;
    const int ldn = (int)round_up(nrhs, 8);
    CFLX_TRY(solve_cache_grow(sc, f, ldn, ch->pk == 0, true));
    CFLX_TRY(solve_seed(sc, f, ldn, nrhs, B, ldb, SolveSeed{false, sc->rows, f.rows, sc->W}));
    if (ch->pk == 0) {  // L Y = B keeping Y_t in Z, then L^T X = Y from Z (signed: R Y = B, R^T X = S Y)
        CFLX_TRY(solve_row_sweep(sc, f, ldn, true, sc->Z, ch->Py, false));
        CFLX_TRY(solve_apply_signs(sc, f, ldn));
        CFLX_TRY(solve_col_sweep(sc, f, ldn, false, Tri::LowerT, sc->X, 1, false));
    }
    return solve_finish(sc, f, ldn, nrhs, X, ldx);
}

const HandleTexts kCholTexts = {
    "requested before a successful cflx_chol_factor, or after cflx_chol_set_local without one",
    "requested before cflx_chol_set_local",
    "refused: the input is already scaled (equed = '%c'); upload it again first"};

// dporfs (UPLO = 'L') on the input A0: A is symmetric, so both kinds of product are cflx_chol_solve's sweeps
RefineOp chol_refine_op(cflx_chol* ch) {
    auto solve = [ch](bool, int n, const double* b, int lb, double* x, int lx) { return chol_sweeps(ch, n, b, lb, x, lx); };
    return RefineOp{*ch, ch->A0, ResidMode::SymLower, true, solve};
}

// LAPACK dpocon on the grid: ||A||_1 of the symmetric input (its stored lower triangle, real tiles only) and the
// Hager-Higham estimate of ||inv(A)||_1, whose products inv(A) x are solves with the factor.
int chol_rcond(cflx_chol* ch, double* rcond_out, double* anorm_out) {
    double anorm = 0.0, ainvnm = 0.0;
    CFLX_TRY(norm1_grid(*ch, ch->A0, true, &anorm));
    if (anorm > 0.0) {
        // every rank runs the estimator on the X of solve_finish, bit-identical on every rank, so every rank makes the
        // same choices and issues the same solves (the same collectives) in the same order; A is symmetric, so both
        // kinds of product are the same solve
        auto apply = [&](int, double* x) { return chol_sweeps(ch, 1, x, 1, x, 1); };
        CFLX_TRY(estimate_inv_norm1(ch->M, apply, &ainvnm));
    }
    *rcond_out = rcond_from(anorm, ainvnm);
    if (anorm_out) *anorm_out = anorm;
    return CFLX_OK;
}

// cflx_chol_equilibrate (dpoequ) and, with pow2, cflx_chol_equilibrate_b (dpoequb), as `who`
int chol_equilibrate(const char* who, cflx_chol* ch, int apply, bool pow2, double* s_out, double* scond_out,
                     double* amax_out, char* equed_out, int* info_out) {
    REFUSE_FOR(who, !ch);
    REFUSE_FOR(who, apply != 0 && apply != 1);
    REFUSE_FOR(who, !info_out);
    if (apply && ch->rbt.in.depth) {
        set_last_error("%s: refused, the input carries a random butterfly transform (cflx_chol_rbt); upload it again first",
                       who);
        return CFLX_ERR_STATE;
    }
    CFLX_TRY(enter(ch, who, NEED_INPUT | (apply ? NEED_UNSCALED : 0u)));
    handle_equil_begin(ch);
    double scond = 0.0, amax = 0.0;
    char equed = 'N';
    int info = 0;
    CFLX_TRY(poequ_grid(*ch, &ch->eq, ch->A0, apply != 0, pow2, s_out, &scond, &amax, &equed, &info));
    CFLX_TRY(handle_equil_end(ch, apply != 0, info, equed, scond, scond, nullptr));
    if (scond_out) *scond_out = scond;
    if (amax_out) *amax_out = amax;
    if (equed_out) *equed_out = equed;
    *info_out = info;
    return CFLX_OK;
}

// The checks of cflx_chol_rbt (`who`) that need no other rank: the rows pair within a rank when 2^d v Px divides N,
// the columns when 2^d v Py does
int chol_rbt_prepare(const char* who, cflx_chol* ch, int depth) {
    REFUSE_FOR(who, depth < 1);
    REFUSE_FOR(who, depth > 4);
    if (ch->rbt.in.depth) {
        set_last_error("%s: refused, the input is already transformed; upload it again first", who);
        return CFLX_ERR_STATE;
    }
    CFLX_TRY(enter(ch, who, NEED_INPUT | NEED_UNSCALED));
    const long long q = ((long long)ch->v * std::lcm(ch->Px, ch->Py)) << depth;
    if (ch->M % q) {
        set_last_error("%s: N = %d is not a multiple of 2^%d v lcm(Px, Py) = %lld; the smallest N that works is %lld: "
                       "pad A with the identity to that order", who, ch->M, depth, q, (ch->M + q - 1) / q * q);
        return CFLX_ERR_UNSUPPORTED;
    }
    return CFLX_OK;
}

// Cholesky.cpp:75-111: the grid chosen for the user, for P >= 1
void chol_auto_grid(int P, int N, int* grid3) {
    if (P == 8 && N < 16384) { grid3[0] = 2; grid3[1] = 2; grid3[2] = 2; }
    else if (P == 32 && N < 8192) { grid3[0] = 4; grid3[1] = 4; grid3[2] = 2; }
    else if (P == 128 && N <= 16384) { grid3[0] = 8; grid3[1] = 8; grid3[2] = 2; }
    else if (P == 512) { grid3[0] = 16; grid3[1] = 16; grid3[2] = 2; }
    else {
        const unsigned pw = (unsigned)std::log2((double)P);
        grid3[0] = pw % 2 == 0 ? 1 << (pw / 2) : (1 << (pw / 2)) * 2;
        grid3[1] = 1 << (pw / 2);
        grid3[2] = 1;
    }
}
// Cholesky.cpp:113-134: the tile size chosen for the user
int chol_auto_tile(int N, int P, int Pz) {
    const double ratio = ((double)N * N * Pz / P) / 1000000.0;
    return ratio < 2.5 ? 128 : (ratio < 30 ? 256 : (ratio < 250 ? 512 : 1024));
}

// o[6] = {N padded to a multiple of v, Kappa, Ml, Nl, nlayr, P} (cflx_chol_dims), refused in the name of `who`
int chol_dims(const char* who, int N, int v, int Px, int Py, int Pz, int* o) {
    REFUSE_FOR(who, N <= 0);
    REFUSE_FOR(who, v <= 0);
    REFUSE_FOR(who, Px <= 0);
    REFUSE_FOR(who, Py <= 0);
    REFUSE_FOR(who, Pz <= 0);
    const int Kappa = (N + v - 1) / v;
    o[0] = Kappa * v; o[1] = Kappa;
    o[2] = ((Kappa + Px - 1) / Px) * v;
    o[3] = ((Kappa + Py - 1) / Py) * v;
    o[4] = v / Pz; o[5] = Px * Py * Pz;
    return CFLX_OK;
}
}  // namespace

// ======================================================================================================== C ABI
extern "C" {

int cflx_chol_auto_grid(int P, int N, int* grid3) {
    REFUSE_IF(P <= 0);
    REFUSE_IF(!grid3);
    chol_auto_grid(P, N, grid3);
    return CFLX_OK;
}
int cflx_chol_auto_tile(int N, int P, int Pz) { return chol_auto_tile(N, P, Pz); }

int cflx_chol_dims(int N, int v, int Px, int Py, int Pz, int* o) {
    REFUSE_IF(!o);
    return chol_dims(__func__, N, v, Px, Py, Pz, o);
}

// CholeskyIO.cpp:100-172: T = lower triangle of R^T R with R = v x v uniform(-1, 1) from rand() after srand(1) (same on
// every rank); every tile of the (lower triangle of the) matrix is T, the global diagonal is 2 * Kappa * max_i sum_j |T_ij|.
// Layers pz != 0 start at zero.  (The reference leaves the upper triangle of its tile buffer unwritten; zeros here.)
// The sequence is glibc's rand() after srand(1), drawn from a state of this call's own (random_r with the 128-byte
// state srand uses): ranks that are threads of one process call this at the same time, and the shared state of rand()
// would deal each of them a different, interleaved R.
int cflx_chol_init_matrix_host(int N, int v, int Px, int Py, int Pz, int rank, double* out) {
    int d[6];
    CFLX_TRY(chol_dims(__func__, N, v, Px, Py, Pz, d));
    REFUSE_IF(rank < 0);
    REFUSE_IF(rank >= Px * Py * Pz);
    REFUSE_IF(!out);
    const int Ml = d[2], Nl = d[3], Kappa = d[1];
    std::fill(out, out + (size_t)Ml * Nl, 0.0);
    if (rank % Pz != 0) return CFLX_OK;
    const int pi = rank / (Py * Pz), pj = (rank / Pz) % Py;
    std::vector<double> R((size_t)v * v), T((size_t)v * v, 0.0);
    alignas(int32_t) char state[128];  // initstate_r keeps its state as int32_t words
    random_data rd{};
    initstate_r(1, state, sizeof(state), &rd);
    for (size_t i = 0; i < (size_t)v * v; ++i) {
        int32_t x = 0;
        random_r(&rd, &x);
        R[i] = (double)x / RAND_MAX * 2 - 1;
    }
    for (int i = 0; i < v; ++i)                 // T = lower(R^T R)  (cblas_dsyrk RowMajor, Lower, Trans)
        for (int j = 0; j <= i; ++j) {
            double s = 0.0;
            for (int k = 0; k < v; ++k) s += R[(size_t)k * v + i] * R[(size_t)k * v + j];
            T[(size_t)i * v + j] = s;
        }
    double mx = -1;
    for (int i = 0; i < v; ++i) {
        double cur = 0.0;
        for (int j = 0; j < v; ++j) cur += std::fabs(T[(size_t)i * v + j]);
        mx = std::max(mx, cur);
    }
    mx = mx * Kappa * 2;
    for (int lti = 0; lti < Ml / v; ++lti)
        for (int ltj = 0; ltj < Nl / v; ++ltj) {
            const int gi = lti * Px + pi, gj = ltj * Py + pj;
            if (gi >= Kappa || gj >= Kappa) continue;
            for (int r = 0; r < v; ++r) std::memcpy(out + (size_t)(lti * v + r) * Nl + (size_t)ltj * v, T.data() + (size_t)r * v, sizeof(double) * v);
            if (gi == gj)
                for (int r = 0; r < v; ++r) out[(size_t)(lti * v + r) * Nl + (size_t)ltj * v + r] = mx;
        }
    return CFLX_OK;
}

int cflx_chol_create(cflx_comm* c, int N, int v, int Px, int Py, int Pz, cflx_chol** out) {
    REFUSE_IF(!c);
    REFUSE_IF(!out);
    REFUSE_IF(N <= 0);
    CFLX_CUDA(cudaSetDevice(c->device));
    if (Px <= 0 || Py <= 0 || Pz <= 0) {
        int g[3];
        chol_auto_grid(c->world_size, N, g);
        Px = g[0]; Py = g[1]; Pz = g[2];
    }
    if (v <= 0) v = chol_auto_tile(N, c->world_size, Pz);
    if (Px * Py * Pz != c->world_size) {
        set_last_error("%s: cholesky grid %dx%dx%d does not match the %d ranks of the communicator", __func__, Px, Py, Pz,
                       c->world_size);
        return CFLX_ERR_ARG;
    }
    if (v % 4 != 0 || v % Pz != 0 || (v / Pz) % 4 != 0 || v > 512 || chol_pick_nb(v) == 0) {
        set_last_error("%s: cholesky tile size v=%d unsupported: need v %% 4 == 0, (v / Pz) %% 4 == 0, v <= 512",
                       __func__, v);
        return CFLX_ERR_UNSUPPORTED;
    }
    int d[6];
    CFLX_TRY(chol_dims(__func__, N, v, Px, Py, Pz, d));
    std::unique_ptr<cflx_chol> ch(new cflx_chol);
    ch->M = d[0]; ch->Nt = d[1]; ch->Ml = d[2]; ch->Nl = d[3]; ch->nlayr = d[4];
    ch->v = v;
    ch->nb = chol_pick_nb(v);
    CFLX_TRY(handle_init(ch.get(), &kCholTexts, c, Px, Py, Pz));
    const size_t vv = (size_t)v * v;
    ch->ldp = chol_panel_ld(ch->Ml);
    ch->ldb = round_up(ch->Nl, 2) + 2;
    CFLX_TRY(ch->PT.alloc((size_t)v * ch->ldp)); CFLX_TRY(ch->LT.alloc((size_t)v * ch->ldp));
    CFLX_TRY(ch->W.alloc((size_t)v * ch->ldp)); CFLX_TRY(ch->G.alloc(2 * (size_t)Px * v * ch->ldp));
    CFLX_TRY(ch->Bc.alloc(2 * (size_t)v * ch->ldb)); CFLX_TRY(ch->D.alloc(vv)); CFLX_TRY(ch->A00.alloc(vv));
    CFLX_TRY(ch->Uinv.alloc(vv)); CFLX_TRY(ch->LinvT.alloc(vv)); CFLX_TRY(ch->acc.alloc(2 + SUMSQ_PARTIALS));
    CFLX_TRY(ch->info.alloc(8));
    if (potrf_tile_scratch(v)) CFLX_TRY(ch->Q.alloc(potrf_tile_scratch(v)));
    cudaMemsetAsync(ch->PT, 0, (size_t)v * ch->ldp * sizeof(double), c->stream);
    cudaMemsetAsync(ch->LT, 0, (size_t)v * ch->ldp * sizeof(double), c->stream);
    cudaMemsetAsync(ch->W, 0, (size_t)v * ch->ldp * sizeof(double), c->stream);
    cudaMemsetAsync(ch->G, 0, 2 * (size_t)Px * v * ch->ldp * sizeof(double), c->stream);
    cudaMemsetAsync(ch->Bc, 0, 2 * (size_t)v * ch->ldb * sizeof(double), c->stream);
    cudaMemsetAsync(ch->A0, 0, (size_t)ch->Ml * ch->Nl * sizeof(double), c->stream);
    cudaMemsetAsync(ch->A00, 0, vv * sizeof(double), c->stream);
    CFLX_TRY(handle_update_setup(ch.get()));
    CFLX_TRY(handle_side_stream(ch.get()));
    CFLX_TRY(ch->ev_col.create(cudaEventDisableTiming));
    CFLX_TRY(ch->ev_panel.create(cudaEventDisableTiming));
    CFLX_TRY(potrf_setup(v));
    CFLX_CUDA(cudaStreamSynchronize(c->stream));
    *out = ch.release();
    return CFLX_OK;
}

// info_out[16] = {N, v, Kappa, Ml, Nl, nlayr, P, Px, Py, Pz, pi, pj, pk, rank, 0, 0}
int cflx_chol_info(const cflx_chol* ch, int* o) {
    REFUSE_IF(!ch);
    REFUSE_IF(!o);
    const int vals[16] = {ch->M, ch->v, ch->Nt, ch->Ml, ch->Nl, ch->nlayr, ch->P, ch->Px, ch->Py, ch->Pz, ch->pi, ch->pj, ch->pk,
                          ch->rank, 0, 0};
    std::memcpy(o, vals, sizeof(vals));
    return CFLX_OK;
}

int cflx_chol_set_local(cflx_chol* ch, const double* host_local) {
    REFUSE_IF(!ch);
    REFUSE_IF(!host_local);
    CFLX_TRY(enter(ch, __func__, 0));
    CFLX_TRY(handle_set_local(ch, host_local));
    ch->rbt.in.depth = 0;
    return CFLX_OK;
}

}  // extern "C"

namespace {
// The factorisation both entry points share (COLLECTIVE), ch->ldlt choosing the signed one: the working copy of the
// input, the look-ahead loop, then *bad = 1 + the first failing column over the grid (0: none), the same on every rank.
// Signed, the last tile's signs (never broadcast) and the counts join the all-reduce of the first failure, into ch->sgn
// and cnt[4].  *ms = device time of the loop.
int chol_factor_run(cflx_chol* ch, float* ms_out, int* bad_out, int* cnt) {
    cflx_comm* c = ch->comm;
    cudaStream_t s = c->stream;
    ch->sv.ready = false;
    ch->factored = false;
    CFLX_TRY(equil_pass_on(&ch->eq, ch->M, false, s));  // the factor carries the input's scaling and transform
    CFLX_TRY(rbt_pass_on(&ch->rbt, ch->M, false, s));
    const int v = ch->v, Py = ch->Py, Ml = ch->Ml, Nl = ch->Nl;
    const int pj = ch->pj;
    CFLX_CUDA(cudaMemcpyAsync(ch->A11, ch->A0, (size_t)Ml * Nl * sizeof(double), cudaMemcpyDeviceToDevice, s));
    CFLX_CUDA(cudaMemsetAsync(ch->info, 0, sizeof(int) * 8, s));
    if (ch->ldlt) {
        CFLX_TRY(ch->sgn.grow(ch->M));
        CFLX_CUDA(cudaMemsetAsync(ch->sgn, 0, sizeof(double) * ch->M, s));  // the last tile's signs are summed
    }
    CFLX_TRY(grid_barrier(c));
    Events<2> loop;
    CFLX_TRY(loop.create());
    CFLX_CUDA(cudaEventRecord(loop[0], s));
    // Look-ahead: the panel pipeline of step k+1 (z-reduce, diagonal Cholesky, solve, piece broadcast -- and every NCCL
    // call of the factorisation) runs on the side stream while the main stream applies the rank-v update of step k; the
    // tile column of step k+1 is updated first so that the side stream can start.
    cudaStream_t sp = ch->side;
    CFLX_CUDA(cudaEventRecord(ch->ev_col[0], s));
    CFLX_CUDA(cudaStreamWaitEvent(sp, ch->ev_col[0], 0));
    CFLX_TRY(panel_step(ch, 0, sp));
    CFLX_CUDA(cudaEventRecord(ch->ev_panel[0], sp));
    for (int k = 0; k + 1 < ch->Nt; ++k) {
        const int b = k & 1, nb1 = (k + 1) & 1;
        CFLX_CUDA(cudaStreamWaitEvent(s, ch->ev_panel[b], 0));             // pieces of step k are in buffer set b
        CFLX_TRY(split_planes(ch, k + 1, k + 1, b, s));                     // (split kinds) both operands
        const int ljn = (k + 1) / Py;                                        // local tile of column k+1 on its owners
        const bool own_next = (pj == (k + 1) % Py);
        if (own_next) CFLX_TRY(update_columns(ch, k + 1, k + 1, b, ch->A11, ljn, ljn + 1, s));
        CFLX_CUDA(cudaEventRecord(ch->ev_col[nb1], s));
        CFLX_CUDA(cudaStreamWaitEvent(sp, ch->ev_col[nb1], 0));
        CFLX_TRY(panel_step(ch, k + 1, sp));
        CFLX_CUDA(cudaEventRecord(ch->ev_panel[nb1], sp));
        CFLX_TRY(update_columns(ch, k + 1, k + 1, b, ch->A11, own_next ? ljn + 1 : 0, Nl / v, s));
    }
    CFLX_CUDA(cudaStreamWaitEvent(s, ch->ev_panel[(ch->Nt - 1) & 1], 0));
    CFLX_CUDA(cudaEventRecord(loop[1], s));
    CFLX_CUDA(cudaEventSynchronize(loop[1]));
    float ms = 0;
    CFLX_CUDA(cudaEventElapsedTime(&ms, loop[0], loop[1]));
    CFLX_CUDA(cudaGetLastError());
    int h[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    CFLX_CUDA(cudaMemcpy(h, ch->info, sizeof(h), cudaMemcpyDeviceToHost));
    int bad = h[1];   // 1 + first failing global column of the diagonal tiles this rank factored, 0 = none
    if (ch->P > 1) {  // the first one over the grid, so that every rank returns the same status and column
        // info[2] is prepared on s, in stream order with the all-reduce that reads it (not an error-handling launch of
        // the factorisation, so it is not counted)
        info_min_operand_kernel<<<1, 1, 0, s>>>(ch->info);
        CFLX_CUDA(cudaGetLastError());
        if (ch->ldlt) CFLX_NCCL(ncclGroupStart());
        CFLX_NCCL(ncclAllReduce(ch->info + 2, ch->info + 2, 1, ncclInt, ncclMin, c->world, s));
        if (ch->ldlt) {  // one owner contributes each sign and each count
            double* last = ch->sgn + (int64_t)(ch->Nt - 1) * v;
            CFLX_NCCL(ncclAllReduce(ch->info + 4, ch->info + 4, 4, ncclInt, ncclSum, c->world, s));
            CFLX_NCCL(ncclAllReduce(last, last, v, ncclDouble, ncclSum, c->world, s));
            CFLX_NCCL(ncclGroupEnd());
        }
        CFLX_CUDA(cudaMemcpyAsync(h, ch->info, sizeof(h), cudaMemcpyDeviceToHost, s));
        CFLX_CUDA(cudaStreamSynchronize(s));
        bad = h[2] == INT_MAX ? 0 : h[2];
    }
    *bad_out = bad;
    ch->low_prec = ch->update.tf32();
    if (cnt) std::memcpy(cnt, h + 4, 4 * sizeof(int));
    *ms_out = ms;
    return CFLX_OK;
}
}  // namespace

extern "C" {

// COLLECTIVE.  parallelCholesky() (Cholesky.cpp:760-921): ms_out = device time of the factorisation loop.
int cflx_chol_factor(cflx_chol* ch, double* ms_out) {
    REFUSE_IF(!ch);
    CFLX_TRY(enter(ch, __func__, NEED_INPUT));
    ch->ldlt = false;
    float ms = 0;
    int bad = 0;
    CFLX_TRY(chol_factor_run(ch, &ms, &bad, nullptr));
    if (bad != 0) {
        set_last_error("%s: the matrix is not positive definite (first non-positive pivot in column %d, counted from 1 like LAPACK dpotrf's info)", __func__, bad);
        return CFLX_ERR_STATE;
    }
    if (ms_out) *ms_out = ms;
    ch->factored = true;
    return CFLX_OK;
}

// COLLECTIVE.  The signed Cholesky A = R S R^T without pivoting (chol_factor_run with ch->ldlt): the factorisation
// completes whatever its pivots; the counts of every rank's diagonal tiles and the first zero pivot come back the same on
// every rank.
int cflx_chol_factor_ldlt(cflx_chol* ch, double tiny, int* nrepl_out, int64_t* inertia_out, int* info_out, double* ms_out) {
    REFUSE_IF(!ch);
    REFUSE_IF(!(tiny >= 0.0));
    REFUSE_IF(!info_out);
    CFLX_TRY(enter(ch, __func__, NEED_INPUT));
    ch->ldlt = true;
    ch->tiny = tiny;
    float ms = 0;
    int bad = 0, cnt[4] = {0, 0, 0, 0};
    const int rc = chol_factor_run(ch, &ms, &bad, cnt);
    if (rc != CFLX_OK) {
        ch->ldlt = false;
        return rc;
    }
    ch->factored = true;
    if (nrepl_out) *nrepl_out = cnt[0];
    if (inertia_out)
        for (int i = 0; i < 3; ++i) inertia_out[i] = cnt[1 + i];
    *info_out = bad;
    if (ms_out) *ms_out = ms;
    return CFLX_OK;
}

// local share of L (Ml x Nl row-major, conflux tile layout; tiles above the diagonal are not meaningful)
int cflx_chol_get_local(cflx_chol* ch, double* L_host) {
    REFUSE_IF(!ch);
    REFUSE_IF(!L_host);
    CFLX_TRY(enter(ch, __func__, NEED_FACTORS));
    CFLX_CUDA(cudaMemcpyAsync(L_host, ch->A11, (size_t)ch->Ml * ch->Nl * sizeof(double), cudaMemcpyDeviceToHost, ch->comm->stream));
    CFLX_CUDA(cudaStreamSynchronize(ch->comm->stream));
    return CFLX_OK;
}

// COLLECTIVE.  ||A - L L^T||_F over the lower triangle (absolute and relative to ||A||_F), on the GPU grid: the update
// sweep is replayed with the stored factor on a copy of the input.  (The reference's checker, examples/cholesky_helper.cpp:
// 183-217, compares against LAPACKE_dpotrf on one node; tests/ do that at small sizes.)
int cflx_chol_validate(cflx_chol* ch, double* abs_out, double* rel_out) {
    REFUSE_IF(!ch);
    CFLX_TRY(enter(ch, __func__, NEED_FACTORS));
    cflx_comm* c = ch->comm;
    cudaStream_t s = c->stream;
    const int v = ch->v, Px = ch->Px, Py = ch->Py, Ml = ch->Ml, Nl = ch->Nl;
    const size_t loc = (size_t)Ml * Nl;
    DevBuf<> Rbuf;
    CFLX_TRY(Rbuf.alloc(loc * sizeof(double)));
    double* R = Rbuf.as<double>();
    // every layer replays with the full contraction on layer 0's factor: only layer 0 holds L, so restrict to pk == 0 by
    // zeroing the other layers' contribution (their A11 holds partial sums, not the factor)
    CFLX_CUDA(cudaMemcpyAsync(R, ch->A0, loc * sizeof(double), cudaMemcpyDeviceToDevice, s));
    const int nlayr_save = ch->nlayr, pk_save = ch->pk;
    for (int t = 0; t < ch->Nt; ++t) {
        int rc = CFLX_OK;
        const int pjt = t % Py;
        const int row0 = first_local_tile(t, ch->pi, Px) * v, n0 = Ml - row0;
        if (ch->pj == pjt && pk_save == 0)
            CFLX_TRY(launch_extract_l_panel_T(ch->A11, Nl, row0, (t / Py) * v, n0, *ch, t, ch->LT, piece_ld(ch, t, ch->pi), s));
        // layer 0 applies the whole contraction, the other layers a zero-length slab (they only take part in the broadcasts)
        ch->nlayr = pk_save == 0 ? v : 0;
        ch->pk = 0;
        if (pk_save == 0) rc = broadcast_and_update(ch, t, t, false, R, s);
        else {
            // participate in the grouped broadcasts only
            ncclResult_t r = ncclGroupStart();
            if (r == ncclSuccess) {
                for (int p = 0; p < Px && r == ncclSuccess; ++p) {
                    const int rows = Ml - first_local_tile(t, p, Px) * v;
                    if (rows <= 0) continue;
                    double* buf = ch->G + (int64_t)p * v * ch->ldp;
                    r = ncclBroadcast(buf, buf, (size_t)v * piece_ld(ch, t, p), ncclDouble, (p * Py + pjt) * ch->Pz, c->world, s);
                }
                const ncclResult_t end = ncclGroupEnd();
                if (r == ncclSuccess) r = end;
            }
            if (r != ncclSuccess) {
                set_last_error("%s: broadcast of step %d -> %s", __func__, t, ncclGetErrorString(r));
                rc = CFLX_ERR_NCCL;
            }
        }
        ch->nlayr = nlayr_save;
        ch->pk = pk_save;
        CFLX_TRY(rc);
    }
    CFLX_CUDA(cudaMemsetAsync(ch->acc, 0, 2 * sizeof(double), s));
    if (pk_save == 0) {   // acc = {the two sums, the per-CTA partials}
        CFLX_TRY(launch_sumsq_lower(R, *ch, ch->acc + 2, ch->acc, s));
        CFLX_TRY(launch_sumsq_lower(ch->A0, *ch, ch->acc + 2, ch->acc + 1, s));
    }
    if (ch->P > 1) CFLX_NCCL(ncclAllReduce(ch->acc, ch->acc, 2, ncclDouble, ncclSum, c->world, s));
    double h[2] = {0, 0};
    CFLX_CUDA(cudaMemcpyAsync(h, ch->acc, sizeof(h), cudaMemcpyDeviceToHost, s));
    if (cudaStreamSynchronize(s) != cudaSuccess) {
        set_last_error("cholesky validation: %s", cudaGetErrorString(cudaGetLastError()));
        return CFLX_ERR_CUDA;
    }
    if (abs_out) *abs_out = std::sqrt(h[0]);
    if (rel_out) *rel_out = std::sqrt(h[0]) / std::sqrt(h[1]);
    return CFLX_OK;
}

// COLLECTIVE.  A X = B with the factor of the last successful cflx_chol_factor (sweeps above); the factor and the input
// are left as they are.
int cflx_chol_solve(cflx_chol* ch, int nrhs, const double* B, int ldb, double* X, int ldx) {
    REFUSE_IF(!ch);
    CFLX_TRY(rhs_args(__func__, nrhs, B, ldb, X, ldx, false));
    CFLX_TRY(enter(ch, __func__, NEED_FACTORS | NEED_FP64));
    return chol_sweeps(ch, nrhs, B, ldb, X, ldx);
}

// COLLECTIVE.  A X = B with B and X distributed like A (solve_local.cu): each block of columns assembled on the device
// and solved by the sweeps of cflx_chol_solve, then scattered into the real rows of X's share.
int cflx_chol_solve_local(cflx_chol* ch, int nrhs, const double* B_local, int ldb, double* X_local, int ldx) {
    REFUSE_IF(!ch);
    SolveLocalArgs a{};
    CFLX_TRY(solve_local_args(__func__, *ch, nrhs, B_local, ldb, X_local, ldx, &a));
    CFLX_TRY(enter(ch, __func__, NEED_FACTORS | NEED_FP64));
    auto solve = [ch](int w, const double* Bk, int ldn, const double** Xk) -> int {
        CFLX_TRY(chol_sweeps(ch, w, Bk, ldn, nullptr, 0));
        *Xk = ch->sv.X;
        return CFLX_OK;
    };
    return solve_local_run(*ch, solve_local_rows(*ch, true), a, solve);
}

// COLLECTIVE.  LAPACK dpotri (UPLO = 'L') on the grid (inverse.cu): the block solves with the identity on the sweeps of
// cflx_chol_solve, the lower tiles of each block column scattered into this rank's share, the rest of it zero.
int cflx_chol_inverse(cflx_chol* ch, double* Ainv_local) {
    REFUSE_IF(!ch);
    CFLX_TRY(enter(ch, __func__, NEED_FACTORS | NEED_FP64));
    if (!ch->sv.ready) CFLX_TRY(chol_solve_prepare(ch));
    return inverse_run(&ch->sv, chol_solve_factor(ch), InvKind::Chol, nullptr, Ainv_local);
}

// COLLECTIVE.  det(A) = prod(l_ii)^2 (det.cu): the diagonal of L from layer 0's A11, its exact-range product squared,
// divided by prod(s)^2 when unscaled.
int cflx_chol_det(cflx_chol* ch, int unscaled, double* logdet_out, double* mant_out, int64_t* exp_out) {
    REFUSE_IF(!ch);
    REFUSE_IF(unscaled != 0 && unscaled != 1);
    CFLX_TRY(enter(ch, __func__, NEED_FACTORS | NEED_FP64));
    const double* s = unscaled && ch->eq.fac.equed == 'Y' ? ch->eq.fac.r.p : nullptr;
    DetResult d{};
    CFLX_TRY(det_grid(*ch, &ch->eq, ch->A11, true, s, nullptr, &d));
    if (ch->ldlt) {  // det = prod(s_i) prod(r_ii)^2: the sign is the parity of the negative signs
        std::vector<double> sg(ch->M);
        CFLX_CUDA(cudaMemcpy(sg.data(), ch->sgn, sizeof(double) * ch->M, cudaMemcpyDeviceToHost));
        if (std::count(sg.begin(), sg.end(), -1.0) & 1) d.mant = -d.mant;
    }
    if (logdet_out) *logdet_out = det_log(d);
    if (mant_out) *mant_out = d.mant;
    if (exp_out) *exp_out = d.exp;
    return CFLX_OK;
}

// COLLECTIVE.  LAPACK dpocon on the grid (chol_rcond).
int cflx_chol_rcond(cflx_chol* ch, double* rcond_out, double* anorm_out) {
    REFUSE_IF(!ch);
    REFUSE_IF(!rcond_out);
    CFLX_TRY(enter(ch, __func__, NEED_FACTORS | NEED_FP64));
    return chol_rcond(ch, rcond_out, anorm_out);
}

// COLLECTIVE.  LAPACK dporfs (UPLO = 'L') on the grid: residuals of the symmetric input from its stored lower triangle
// (refine.cu), corrections and both kinds of estimator product by cflx_chol_solve's sweeps.
int cflx_chol_refine(cflx_chol* ch, int nrhs, const double* B, int ldb, double* X, int ldx, double* ferr_out,
                     double* berr_out) {
    REFUSE_IF(!ch);
    CFLX_TRY(rhs_args(__func__, nrhs, B, ldb, X, ldx, true));
    CFLX_TRY(enter(ch, __func__, NEED_FACTORS | NEED_FP64));
    return refine_run(&ch->sv.rf, chol_refine_op(ch), nrhs, B, ldb, X, ldx, ferr_out, berr_out);
}

// COLLECTIVE.  LAPACK dporfsx (UPLO = 'L') on the grid: dpocon, then refine_x_run with the symmetric residual and the
// scales s of the solution's rows (equed Y).  A successful factorisation has no zero pivot.
int cflx_chol_refine_x(cflx_chol* ch, int nrhs, const double* B, int ldb, double* X, int ldx, double* rcond_out,
                       double* berr_out, double* err_bnds_norm_out, double* err_bnds_comp_out, int* info_out) {
    REFUSE_IF(!ch);
    CFLX_TRY(rhs_args(__func__, nrhs, B, ldb, X, ldx, true));
    REFUSE_IF(!err_bnds_norm_out);
    REFUSE_IF(!info_out);
    CFLX_TRY(enter(ch, __func__, NEED_FACTORS | NEED_FP64));
    double rcond = 0.0;
    CFLX_TRY(chol_rcond(ch, &rcond, nullptr));
    if (rcond_out) *rcond_out = rcond;
    const EquilRecord& eq = ch->eq.fac;
    return refine_x_run(&ch->sv.rf, chol_refine_op(ch), nrhs, B, ldb, X, ldx, eq.equed == 'Y' ? eq.r.p : nullptr, rcond,
                        err_bnds_comp_out != nullptr, berr_out, err_bnds_norm_out, err_bnds_comp_out, info_out);
}

// COLLECTIVE.  LAPACK dpoequ (+ dlaqsy, UPLO = 'L', when apply) on the input A0 (equil.cu); drops the factorisation and
// the solve cache, as cflx_chol_set_local does.
int cflx_chol_equilibrate(cflx_chol* ch, int apply, double* s_out, double* scond_out, double* amax_out, char* equed_out,
                          int* info_out) {
    return chol_equilibrate(__func__, ch, apply, false, s_out, scond_out, amax_out, equed_out, info_out);
}

// COLLECTIVE.  LAPACK dpoequb (+ dlaqsy when apply): cflx_chol_equilibrate with the scales rounded to powers of two.
int cflx_chol_equilibrate_b(cflx_chol* ch, int apply, double* s_out, double* scond_out, double* amax_out,
                            char* equed_out, int* info_out) {
    return chol_equilibrate(__func__, ch, apply, true, s_out, scond_out, amax_out, equed_out, info_out);
}

// COLLECTIVE.  LAPACK dposvx after a successful factorisation, with the scaling the factor carries: B scaled by s,
// dpocon, the solve, dporfs, X unscaled by s and ferr divided by scond.
int cflx_chol_svx(cflx_chol* ch, int nrhs, const double* B, int ldb, double* X, int ldx, double* rcond_out,
                  double* ferr_out, double* berr_out, char* equed_out, int* info_out) {
    REFUSE_IF(!ch);
    CFLX_TRY(rhs_args(__func__, nrhs, B, ldb, X, ldx, true));
    REFUSE_IF(!rcond_out);
    REFUSE_IF(!info_out);
    CFLX_TRY(enter(ch, __func__, NEED_FACTORS | NEED_FP64));
    const EquilRecord& eq = ch->eq.fac;
    const double* s = eq.equed == 'Y' ? eq.r.p : nullptr;
    if (equed_out) *equed_out = eq.equed;
    double rcond = 0.0;
    CFLX_TRY(chol_rcond(ch, &rcond, nullptr));
    *rcond_out = rcond;
    return svx_run(&ch->eq, &ch->sv.rf, chol_refine_op(ch), nrhs, B, ldb, X, ldx, ferr_out, berr_out, s, s, eq.rowcnd,
                   rcond, info_out);
}

// COLLECTIVE.  LAPACK dposvxx after a successful factorisation, with the scaling the factor carries: dla_porpvgrw of the
// stored lower triangles of the input and of L, dpocon, B scaled by s, the solve, dporfsx's refinement as
// cflx_chol_refine_x runs it, X unscaled by s.
int cflx_chol_svxx(cflx_chol* ch, int nrhs, const double* B, int ldb, double* X, int ldx, double* rcond_out,
                   double* rpvgrw_out, double* berr_out, double* err_bnds_norm_out, double* err_bnds_comp_out,
                   char* equed_out, int* info_out) {
    REFUSE_IF(!ch);
    CFLX_TRY(rhs_args(__func__, nrhs, B, ldb, X, ldx, true));
    REFUSE_IF(!rcond_out);
    REFUSE_IF(!err_bnds_norm_out);
    REFUSE_IF(!info_out);
    CFLX_TRY(enter(ch, __func__, NEED_FACTORS | NEED_FP64));
    const EquilRecord& eq = ch->eq.fac;
    const double* s = eq.equed == 'Y' ? eq.r.p : nullptr;
    if (equed_out) *equed_out = eq.equed;
    std::vector<double> h;
    CFLX_TRY(growth_cols_grid(*ch, &ch->eq, true, ch->A11, ch->A0, ch->M, h));
    if (rpvgrw_out) *rpvgrw_out = rpvgrw_cols(h, ch->M, ch->M);
    double rcond = 0.0;
    CFLX_TRY(chol_rcond(ch, &rcond, nullptr));
    *rcond_out = rcond;
    return svxx_run(&ch->eq, &ch->sv.rf, chol_refine_op(ch), nrhs, B, ldb, X, ldx, s, s, s, rcond,
                    err_bnds_comp_out != nullptr, berr_out, err_bnds_norm_out, err_bnds_comp_out, info_out);
}

// COLLECTIVE.  LAPACK dsposv on the grid: the input factored with the TF32 trailing update (prec 1: one term, 3: three),
// then mixed_run's refinement in FP64 on the stored lower triangle of A0.  When the low-precision factorisation meets a
// non-positive pivot (iter -3) or the loop does not converge (-31), the input is factored again in FP64 and solved, as
// cflx_chol_factor + cflx_chol_solve do; the handle then holds that FP64 factor, or none when the FP64 factorisation
// fails too (CFLX_ERR_STATE as cflx_chol_factor, with *iter_out set).
int cflx_chol_sv_mixed(cflx_chol* ch, int prec, int nrhs, const double* B, int ldb, double* X, int ldx, int itmax,
                       int* iter_out, double* berr_out, double* ms_out) {
    REFUSE_IF(!ch);
    REFUSE_IF(prec != CFLX_PREC_TF32 && prec != CFLX_PREC_TF32X3);
    REFUSE_IF(!iter_out);
    CFLX_TRY(rhs_args(__func__, nrhs, B, ldb, X, ldx, true));
    CFLX_TRY(enter(ch, __func__, NEED_INPUT | NEED_UNSCALED));
    if (ch->rbt.in.depth) {
        set_last_error("%s: refused, the input carries a random butterfly transform (cflx_chol_rbt); upload it again first",
                       __func__);
        return CFLX_ERR_STATE;
    }
    ch->ldlt = false;
    float ms = 0;
    int bad = 0;
    CFLX_TRY(ch->update.with_tf32(prec, [&] { return chol_factor_run(ch, &ms, &bad, nullptr); }));
    double anorm = 0.0;  // the infinity-norm of the symmetric matrix is its 1-norm
    CFLX_TRY(norm1_grid(*ch, ch->A0, true, &anorm));
    int iter = MIXED_LOW_PREC_FAILED;
    if (bad == 0) {
        ch->factored = true;
        CFLX_TRY(mixed_run(&ch->sv.rf, chol_refine_op(ch), anorm, itmax > 0 ? itmax : MIXED_ITMAX, nrhs, B, ldb, X, ldx,
                           &iter, berr_out));
    }
    *iter_out = iter;
    double total = ms;
    if (iter < 0) {
        CFLX_TRY(chol_factor_run(ch, &ms, &bad, nullptr));
        total += ms;
        if (ms_out) *ms_out = total;
        if (bad != 0) {
            set_last_error("%s: the matrix is not positive definite (first non-positive pivot of the FP64 factorisation in "
                           "column %d, counted from 1 like LAPACK dpotrf's info)", __func__, bad);
            return CFLX_ERR_STATE;
        }
        ch->factored = true;
        CFLX_TRY(chol_sweeps(ch, nrhs, B, ldb, X, ldx));
        if (berr_out) CFLX_TRY(mixed_berr(&ch->sv.rf, chol_refine_op(ch), anorm, nrhs, B, ldb, X, ldx, berr_out));
    }
    if (ms_out) *ms_out = total;
    return CFLX_OK;
}

// The signs S of the last factorisation: those of cflx_chol_factor_ldlt, or all +1 after cflx_chol_factor
int cflx_chol_get_signs(cflx_chol* ch, double* s_out) {
    REFUSE_IF(!ch);
    REFUSE_IF(!s_out);
    CFLX_TRY(enter(ch, __func__, NEED_FACTORS));
    if (!ch->ldlt) {
        std::fill(s_out, s_out + ch->M, 1.0);
        return CFLX_OK;
    }
    CFLX_CUDA(cudaMemcpy(s_out, ch->sgn, sizeof(double) * ch->M, cudaMemcpyDeviceToHost));
    return CFLX_OK;
}

// the input share as the factorisations read it (after an equilibration that scaled it, after cflx_chol_rbt)
int cflx_chol_get_input(cflx_chol* ch, double* A_host) {
    REFUSE_IF(!ch);
    REFUSE_IF(!A_host);
    CFLX_TRY(enter(ch, __func__, NEED_INPUT));
    CFLX_CUDA(cudaMemcpyAsync(A_host, ch->A0, (size_t)ch->Ml * ch->Nl * sizeof(double), cudaMemcpyDeviceToHost, ch->comm->stream));
    CFLX_CUDA(cudaStreamSynchronize(ch->comm->stream));
    return CFLX_OK;
}

// COLLECTIVE.  A0 <- W = U^T A0 U on every rank's share (rbt.cu), after the ranks agreed on depth and seed with one world
// all-reduce, so that a refusal anywhere is a refusal everywhere: first the symmetric completion of the stored lower
// triangle (sym_mirror), since a butterfly row pair mixes both triangles, then the two-sided transform with V = U.  Every
// layer transforms its own share (the transform is linear).  The factor and the solve cache are dropped.  The input
// carries the transform only once both passes succeeded; a failure after the mirror began leaves no input at all (a
// half-transformed share must be uploaded again).
int cflx_chol_rbt(cflx_chol* ch, int depth, uint64_t seed, double* u_out) {
    REFUSE_IF(!ch);
    CFLX_TRY(enter(ch, __func__, 0));  // the device of world_agree, whatever chol_rbt_prepare finds
    const int rc = chol_rbt_prepare(__func__, ch, depth);
    bool same = false;
    CFLX_TRY(world_agree(ch, rc == CFLX_OK, {seed, (unsigned long long)depth}, &same));
    if (rc != CFLX_OK) return rc;
    if (!same) {
        set_last_error("%s: the ranks passed different depths or seeds, or another rank refused its arguments", __func__);
        return CFLX_ERR_ARG;
    }
    const int M = ch->M;
    const size_t n = (size_t)depth * M;
    std::vector<double> r(n), sc(2 * n);
    rbt_multipliers(M, depth, seed, 0, r.data());
    if (u_out) std::memcpy(u_out, r.data(), sizeof(double) * n);
    rbt_scales(r.data(), n, sc.data());
    std::memcpy(sc.data() + n, sc.data(), sizeof(double) * n);  // the record's V is U
    cudaStream_t s = ch->comm->stream;
    ch->factored = false;
    ch->sv.ready = false;
    RbtRecord& in = ch->rbt.in;
    int rc2 = sym_mirror(*ch, ch->A0);
    if (rc2 == CFLX_OK) rc2 = rbt_record_set(&in, depth, seed, sc.data(), M, s);
    if (rc2 == CFLX_OK) rc2 = launch_rbt(RbtOp::W, ch->A0, ch->Nl, *ch, ch->Nl, INT_MAX, depth, in.s, in.s, s);
    if (rc2 == CFLX_OK && cudaStreamSynchronize(s) != cudaSuccess) {  // sc is a host temporary
        set_last_error("%s: %s", __func__, cudaGetErrorString(cudaGetLastError()));
        rc2 = CFLX_ERR_CUDA;
    }
    if (rc2 != CFLX_OK) {
        in.depth = 0;
        ch->have_input = false;
    }
    return rc2;
}

// COLLECTIVE.  A X = B through the transformed system the factor represents: X = U inv(W) U^T B, with dporfs on the
// transformed system when refine (svx_tail with the butterflies as its row transforms).
int cflx_chol_rbt_solve(cflx_chol* ch, int nrhs, const double* B, int ldb, double* X, int ldx, int refine,
                        double* ferr_out, double* berr_out) {
    REFUSE_IF(!ch);
    REFUSE_IF(refine != 0 && refine != 1);
    CFLX_TRY(rhs_args(__func__, nrhs, B, ldb, X, ldx, true));
    CFLX_TRY(enter(ch, __func__, NEED_FACTORS | NEED_FP64));
    if (!ch->rbt.fac.depth) {
        set_last_error("%s: the factor carries no random butterfly transform (cflx_chol_rbt before the factorisation)",
                       __func__);
        return CFLX_ERR_STATE;
    }
    const RefineOp op = chol_refine_op(ch);
    auto refine_step = [&](const double* dB, int lb, double* dX, int lx) {
        return refine ? refine_run(&ch->sv.rf, op, nrhs, dB, lb, dX, lx, ferr_out, berr_out) : CFLX_OK;
    };
    return svx_tail(&ch->eq, op, nrhs, B, ldb, X, ldx, rbt_rows(*ch, RbtOp::UT), rbt_rows(*ch, RbtOp::U), refine_step);
}

// Not collective.  U^T (op 0) or U (op 1) of the factor's transform on the rows of this rank's right-hand side share.
int cflx_chol_rbt_apply_local(cflx_chol* ch, int op, int nrhs, double* B_local, int ldb) {
    REFUSE_IF(!ch);
    REFUSE_IF(op != 0 && op != 1);
    REFUSE_IF(nrhs < 1);
    REFUSE_IF(!B_local);
    REFUSE_IF(ldb < rhs_local_cols(nrhs, ch->v, ch->Py));
    return rbt_apply_local(__func__, "cflx_chol_rbt", ch, op ? RbtOp::U : RbtOp::UT, nrhs, B_local, ldb);
}

int cflx_chol_launch_count(cflx_chol* ch, int64_t* count_out, int reset) {
    REFUSE_IF(!ch);
    REFUSE_IF(!count_out);
    return handle_launch_count(ch, count_out, reset);
}

void cflx_chol_destroy(cflx_chol* ch) { delete ch; }

}  // extern "C"

cflx_chol::~cflx_chol() {
    cudaSetDevice(comm->device);
    if (j_comm.c) ncclCommDestroy(j_comm.c);
    grid_free(this);
}
