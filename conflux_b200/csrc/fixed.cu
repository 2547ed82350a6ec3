// conflux_b200/csrc/fixed.cu -- the kernels of the LU in a prescribed row order (cflx_lu_factor_fixed): the unpivoted
// LU of one v x v diagonal block with the tiny-pivot rule, the row-locate map of a step's prescribed rows, and the
// operand of the end-of-factorisation minimum over the first zero pivot.
#include <climits>

#include "lu_state.h"

namespace cflx {
namespace {
constexpr int FB = 32;        // column block of the right-looking tile LU
constexpr int FP = FB + 2;    // pitch of the block column in shared memory (even: 16-byte rows for the double2 reads)
constexpr int FTHREADS = 512;  // 128 registers per thread: one row (column) of a block in registers
constexpr int QB = 128;        // block column of the blocked tile driver

// Unpivoted LU of ONE n x n block by ONE CTA, in place, right-looking over 32-column blocks.
//   A    in/out: the block (leading dimension lda), out: L\U (unit L below the diagonal, U on and above it)
//   Ac   out (may be null): a contiguous n x n copy of L\U;  ATc out (may be null): its contiguous transpose
//   rec  (may be null): rec[0] += the pivots replaced; rec[1] = col0 + 1 + the first exactly zero pivot's column, when
//        rec[1] is 0 and there is one
// A pivot u with |u| < tiny becomes copysign(tiny, u), +tiny for +-0; with tiny == 0 nothing is replaced.  The block
// column being factored sits in `Ls` ([n][FP]: dynamic shared memory, or gpanel when n is too large for it).  Every
// sum runs in a fixed order: the same bits on every call.
__global__ void __launch_bounds__(FTHREADS) getrf_nopiv_block_kernel(double* __restrict__ A, int lda, int v, double tiny,
                                                                     double* __restrict__ Ac, double* __restrict__ ATc,
                                                                     int* __restrict__ rec, int col0,
                                                                     double* __restrict__ gpanel) {
    extern __shared__ double smem_fixed[];
    double* Ls = gpanel ? gpanel : smem_fixed;
    __shared__ int s_nrepl, s_zero;
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    constexpr int NW = FTHREADS / 32;
    if (t == 0) s_nrepl = 0, s_zero = 0;
    __syncthreads();
    for (int jb = 0; jb < v; jb += FB) {
        const int nb = min(FB, v - jb), rows = v - jb, m = rows - nb;
        // the block column, rows jb.., zeros beyond its nb columns
        for (int e = t; e < rows * FB; e += FTHREADS) {
            const int r = e / FB, c = e % FB;
            Ls[r * FP + c] = c < nb ? A[(size_t)(jb + r) * lda + jb + c] : 0.0;
        }
        __syncthreads();
        if (warp == 0) {  // the nb x nb diagonal block, lane = row, the row in registers, row c by shuffles
            double a[FB];
#pragma unroll
            for (int c = 0; c < FB; ++c) a[c] = lane < nb ? Ls[lane * FP + c] : 0.0;  // Ls holds rows < v - jb only
#pragma unroll
            for (int c = 0; c < FB; ++c) {
                if (c < nb) {
                    double d = __shfl_sync(0xffffffffu, a[c], c);
                    const bool repl = fabs(d) < tiny;
                    if (repl) d = d == 0.0 ? tiny : copysign(tiny, d);
                    if (lane == 0) {
                        s_nrepl += repl;
                        if (d == 0.0 && s_zero == 0) s_zero = col0 + jb + c + 1;
                    }
                    if (lane == c) a[c] = d;
                    else if (lane > c) a[c] = a[c] / d;
#pragma unroll
                    for (int c2 = c + 1; c2 < FB; ++c2) {
                        const double u = __shfl_sync(0xffffffffu, a[c2], c);  // U[c][c2]
                        if (lane > c) a[c2] = fma(-a[c], u, a[c2]);
                    }
                }
            }
            if (lane < nb) {
#pragma unroll
                for (int c = 0; c < FB; ++c)
                    if (c < nb) Ls[lane * FP + c] = a[c];
            }
        }
        __syncthreads();
        // rows below the diagonal block: L21 = A21 inv(U11), in place in Ls, one row per thread
        for (int r = nb + t; r < rows; r += FTHREADS) {
            double x[FB];
#pragma unroll
            for (int c = 0; c < FB; ++c) x[c] = Ls[r * FP + c];
#pragma unroll
            for (int c = 0; c < FB; ++c) {
                if (c < nb) {
                    double s = x[c];
#pragma unroll
                    for (int q = 0; q < c; ++q) s = fma(-x[q], Ls[q * FP + c], s);
                    x[c] = s / Ls[c * FP + c];
                }
            }
#pragma unroll
            for (int c = 0; c < FB; ++c)
                if (c < nb) Ls[r * FP + c] = x[c];
        }
        // columns right of it: U12 = inv(L11) A12 (unit L11), in place in A, one column per thread
        for (int j = jb + nb + t; j < v; j += FTHREADS) {
            double y[FB];
#pragma unroll
            for (int r = 0; r < FB; ++r) {
                if (r < nb) {
                    double s = A[(size_t)(jb + r) * lda + j];
#pragma unroll
                    for (int q = 0; q < r; ++q) s = fma(-Ls[r * FP + q], y[q], s);
                    y[r] = s;
                    A[(size_t)(jb + r) * lda + j] = s;
                }
            }
        }
        __syncthreads();
        // the factored block column back into A (columns jb.., the trailing update below touches columns >= jb + nb)
        for (int e = t; e < rows * nb; e += FTHREADS) {
            const int r = e / nb, c = e % nb;
            A[(size_t)(jb + r) * lda + jb + c] = Ls[r * FP + c];
        }
        // trailing block: A22 -= L21 U12; a warp takes 16 rows x 32 columns, lane = column, U12's column in registers
        if (m > 0) {
            const int ct = (m + 31) / 32, rg = (m + 15) / 16;
            for (int w = warp; w < ct * rg; w += NW) {
                const int ti = w / ct, j = jb + nb + (w % ct) * 32 + lane;
                const bool jok = j < v;
                double u[FB];
#pragma unroll
                for (int c = 0; c < FB; ++c) u[c] = (jok && c < nb) ? A[(size_t)(jb + c) * lda + j] : 0.0;
#pragma unroll 1
                for (int q = 0; q < 16; ++q) {
                    const int r = nb + ti * 16 + q;
                    if (r >= rows) break;
                    const double* lp = Ls + r * FP;
                    double s = 0.0;
#pragma unroll
                    for (int c = 0; c < FB; c += 2) {
                        const double2 l2 = *reinterpret_cast<const double2*>(lp + c);
                        s = fma(l2.x, u[c], s);
                        s = fma(l2.y, u[c + 1], s);
                    }
                    if (jok) A[(size_t)(jb + r) * lda + j] -= s;
                }
            }
        }
        __syncthreads();
    }
    if (Ac || ATc) {
        for (int e = t; e < v * v; e += FTHREADS) {
            const int i = e / v, c = e % v;
            const double x = A[(size_t)i * lda + c];
            if (Ac) Ac[e] = x;
            if (ATc) ATc[(size_t)c * v + i] = x;
        }
    }
    if (t == 0 && rec) {
        rec[0] += s_nrepl;
        if (rec[1] == 0 && s_zero) rec[1] = s_zero;
    }
}

// pos[i] = the active panel position of global row g = rows[i] on this rank (grid row pi of Px), or n_old where another
// grid row owns it: original local row (g / (v Px)) v + g % v, now at local row igri[.] (after the pushes of the
// earlier steps), minus the fnpr rows already promoted
__global__ void fixed_locate_kernel(const int* __restrict__ rows, int v, int Px, int pi, int fnpr, int n_old,
                                    const int* __restrict__ igri, int* __restrict__ pos) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= v) return;
    const int g = rows[i];
    pos[i] = ((g / v) % Px == pi) ? igri[(g / (v * Px)) * v + g % v] - fnpr : n_old;
}

// rec[2] = rec[1], or INT_MAX when this rank factored no exactly zero pivot: the operand of the ncclMin over the world
__global__ void fixed_info_operand_kernel(int* rec) { rec[2] = rec[1] ? rec[1] : INT_MAX; }

size_t tile_smem(int v) { return (size_t)v * FP * sizeof(double); }
}  // namespace

bool getrf_nopiv_blocked(int v) { return v % QB == 0 && v >= 2 * QB; }

size_t getrf_nopiv_scratch(int v, bool blocked) {
    if (blocked) return (size_t)4 * QB * QB + (size_t)4 * QB * v;
    int dev = 0, opt = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&opt, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess) {
        cudaGetLastError();
        opt = 0;
    }
    return tile_smem(v) + 64 <= (size_t)opt ? 0 : (size_t)v * FP;
}

// One launch of the one-CTA kernel on the n x n window A (lda); the block column in shared memory, or in gpanel
int block_lu(double* A, int lda, int n, double tiny, double* Ac, double* ATc, int* rec, int col0, double* gpanel,
             cudaStream_t s) {
    static PerDeviceMax cfg;
    const size_t smem = gpanel ? 0 : tile_smem(n);
    if (cfg.raise(smem))
        CFLX_CUDA(cudaFuncSetAttribute(getrf_nopiv_block_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    getrf_nopiv_block_kernel<<<1, FTHREADS, smem, s>>>(A, lda, n, tiny, Ac, ATc, rec, col0, gpanel);
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}

// The one-CTA kernel alone is far too slow for a 256 or 512 tile (one SM does all of its O(v^3) work, and the search it
// replaces takes ~0.6 ms), so with `blocked` the tile is factored in 128-wide block columns, as potrf_tile does: the
// 128 x 128 diagonal block on the one-CTA kernel, the block column below it and the block row right of it by the TRSMs
// with its inverted diagonal blocks, and the rest of the tile by one rank-128 update on the FP64 DMMA GEMM.
int launch_getrf_nopiv_tile(const double* Bt, int v, double tiny, double* A, double* AT, const int* tags_in, int* tags_out,
                            int* rec, int col0, bool blocked, double* scratch, cudaStream_t s, int64_t* launches) {
    CFLX_TRY(launch_extract_panel_T(Bt, v, 0, 0, v, v, A, v, s));  // A[i][c] = Bt[c][i]
    ++*launches;
    if (tags_out) CFLX_CUDA(cudaMemcpyAsync(tags_out, tags_in, sizeof(int) * v, cudaMemcpyDeviceToDevice, s));
    if (!blocked) {
        CFLX_TRY(block_lu(A, v, v, tiny, nullptr, AT, rec, col0, scratch, s));
        ++*launches;
        return CFLX_OK;
    }
    double* Dc = scratch;                  // [QB][QB]  L\U of the current diagonal block, contiguous
    double* DcT = Dc + QB * QB;            // [QB][QB]  its transpose
    double* Ui = DcT + QB * QB;            // [QB][QB]  inverse of its U
    double* Li = Ui + QB * QB;             // [QB][QB]  inverse of its unit L, transposed
    double* XT0 = Li + QB * QB;            // [QB][v]   block column below it, transposed
    double* XT = XT0 + (size_t)QB * v;     // [QB][v]   ... L21^T after the solve
    double* R = XT + (size_t)QB * v;       // [QB][v]   block row right of it
    double* U = R + (size_t)QB * v;        // [QB][v]   ... U12 after the solve
    for (int jb = 0; jb < v; jb += QB) {
        const int m = v - jb - QB;
        double* Djj = A + (size_t)jb * v + jb;
        CFLX_TRY(block_lu(Djj, v, QB, tiny, Dc, DcT, rec, col0 + jb, nullptr, s));
        ++*launches;
        if (m <= 0) break;
        CFLX_TRY(launch_diag_inverses(Dc, QB, QB, Ui, Li, s));
        CFLX_TRY(launch_extract_panel_T(A, v, jb + QB, jb, m, QB, XT0, m, s));
        CFLX_TRY(trsm_right_upper_T(Dc, Ui, QB, QB, XT0, XT, m, m, s));          // L21 = A21 inv(U11)
        CFLX_TRY(launch_store_panel_T(A, v, jb + QB, jb, m, QB, XT, m, s));
        CFLX_CUDA(cudaMemcpy2DAsync(R, (size_t)m * sizeof(double), Djj + QB, (size_t)v * sizeof(double),
                                    (size_t)m * sizeof(double), QB, cudaMemcpyDeviceToDevice, s));
        CFLX_TRY(trsm_left_lower_unit(DcT, Li, QB, QB, R, U, m, m, s));           // U12 = inv(L11) A12
        CFLX_CUDA(cudaMemcpy2DAsync(Djj + QB, (size_t)v * sizeof(double), U, (size_t)m * sizeof(double),
                                    (size_t)m * sizeof(double), QB, cudaMemcpyDeviceToDevice, s));
        GemmArgs g{};                                                             // A22 -= L21 U12
        g.M = m; g.N = m; g.K = QB;
        g.AT = XT; g.ldat = m;
        g.B = U; g.ldb = m;
        g.C = A + (size_t)(jb + QB) * v + jb + QB; g.ldc = v;
        g.D = A + (size_t)(jb + QB) * v + jb + QB; g.ldd = v;
        g.alpha = -1.0; g.beta = 1.0;
        CFLX_TRY(launch_gemm_tn(g, s));
        *launches += 6;
    }
    if (AT) {
        CFLX_TRY(launch_extract_panel_T(A, v, 0, 0, v, v, AT, v, s));
        ++*launches;
    }
    return CFLX_OK;
}

int launch_fixed_locate(const int* rows, int v, int Px, int pi, int fnpr, int n_old, const int* igri, int* pos,
                        cudaStream_t s) {
    fixed_locate_kernel<<<(v + 255) / 256, 256, 0, s>>>(rows, v, Px, pi, fnpr, n_old, igri, pos);
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}

int launch_fixed_info_operand(int* rec, cudaStream_t s) {
    fixed_info_operand_kernel<<<1, 1, 0, s>>>(rec);
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}
}  // namespace cflx
