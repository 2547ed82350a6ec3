// conflux_b200/csrc/rows.cu -- HBM-bound row/panel movement kernels of the LU step (K2-K4, K8, K9 of SURVEY.md 2.3).
// All of them are pure data movement: coalesced, 128-bit where the layout allows, grids sized by the data.
//
// Reference call sites replaced (relative to /root/reference/src/conflux/lu):
//   conflux_opt.hpp:620-622,698-705   panel extract (parallel_mcopy + prepend_column)  -> extract_panel_T
//   utils.hpp:85-116                  inverse_permute_rows (winner extraction)          -> gather_winners
//   conflux_opt.cpp:74-148            g2lnoTile + analyze_pivots                        -> plan_moves (one CTA)
//   conflux_opt.hpp:176-218,1041-1090 push_pivots_up on A11Buff / A10Buff / gri         -> push_phase1..3,
//                                                                                         compact_panel, update_gri
//   conflux_opt.hpp:1137-1147         pivot-row extract into A01BuffTemp                -> fused into push_phase1
//   conflux_opt.hpp:1680-1771         validation stores of L / U / A00                  -> store_panel_T,
//                                                                                         store_u_rows, store_diag
#include <algorithm>

#include "common.cuh"
#include "kernels.h"

namespace cflx {

namespace {

// ---------------------------------------------------------------- transposing panel copies
__global__ void extract_panel_T_kernel(const double* __restrict__ A, int64_t lda, int64_t row0, int64_t col0, int n,
                                       int v, double* __restrict__ PT, int64_t ldp) {
    __shared__ double tile[32][33];
    const int r0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    for (int dy = threadIdx.y; dy < 32; dy += blockDim.y) {
        const int r = r0 + dy, c = c0 + threadIdx.x;
        if (r < n && c < v) tile[dy][threadIdx.x] = A[(row0 + r) * lda + col0 + c];
    }
    __syncthreads();
    for (int dy = threadIdx.y; dy < 32; dy += blockDim.y) {
        const int c = c0 + dy, r = r0 + threadIdx.x;
        if (r < n && c < v) PT[(int64_t)c * ldp + r] = tile[threadIdx.x][dy];
    }
}
__global__ void store_panel_T_kernel(double* __restrict__ A, int64_t lda, int64_t row0, int64_t col0, int n, int v,
                                     const double* __restrict__ LT, int64_t ldp) {
    __shared__ double tile[32][33];
    const int r0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    for (int dy = threadIdx.y; dy < 32; dy += blockDim.y) {
        const int c = c0 + dy, r = r0 + threadIdx.x;
        if (r < n && c < v) tile[dy][threadIdx.x] = LT[(int64_t)c * ldp + r];
    }
    __syncthreads();
    for (int dy = threadIdx.y; dy < 32; dy += blockDim.y) {
        const int r = r0 + dy, c = c0 + threadIdx.x;
        if (r < n && c < v) A[(row0 + r) * lda + col0 + c] = tile[threadIdx.x][dy];
    }
}

// ---------------------------------------------------------------- winners of a pivot search
__global__ void gather_winners_kernel(const double* __restrict__ PT, int64_t ldp, const int* __restrict__ tags,
                                      int n_valid, const int* __restrict__ perm, int v, double* __restrict__ out,
                                      int64_t ldo, int* __restrict__ out_tags, int dst0) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (int64_t)v * v) return;
    const int c = (int)(e / v), i = (int)(e % v);
    const int src = perm[i];
    out[(int64_t)c * ldo + dst0 + i] = src < n_valid ? PT[(int64_t)c * ldp + src] : 0.0;
    if (c == 0) out_tags[dst0 + i] = src < n_valid ? tags[src] : 0;
}
__global__ void gather_a00_kernel(const double* __restrict__ W, int64_t ldw, const int* __restrict__ perm, int v, int nb,
                                  double* __restrict__ A00, double* __restrict__ A00T) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (int64_t)v * v) return;
    const int i = (int)(e / v), c = (int)(e % v);
    double val;
    if (nb <= 0 || c < (i / nb) * nb) {  // nb <= 0: the search kernel emitted nothing, every entry comes from W
        val = W[(int64_t)c * ldw + perm[i]];
        A00[e] = val;
    } else {
        val = A00[e];
    }
    A00T[(int64_t)c * v + i] = val;
}

// ---------------------------------------------------------------- step-2 planner (one CTA)
__global__ void __launch_bounds__(256) plan_moves_kernel(const int* __restrict__ gpivots, int v, int Px, int pi, int fnpr,
                                                         int Ml, const int* __restrict__ igri, MovePlan plan) {
    extern __shared__ int sm[];
    int* mine = sm;        // [v] 1 if pivot i lives on this rank
    int* prow = sm + v;    // [v] local row of my pivot (by rank)
    __shared__ int s_npiv, s_nel;
    const int t = threadIdx.x, T = blockDim.x;
    for (int i = t; i < v; i += T) mine[i] = ((gpivots[i] / v) % Px == pi) ? 1 : 0;
    for (int r = fnpr + t; r < Ml; r += T) plan.rowsrc[r] = r;
    __syncthreads();
    for (int i = t; i < v; i += T) {
        int rank = 0;
        for (int j = 0; j < i; ++j) rank += mine[j];
        if (mine[i]) {
            const int g = gpivots[i];
            const int lidx = (g / (v * Px)) * v + g % v;  // original local row of global row g on its owner
            const int lrow = igri[lidx];
            plan.cur_piv[rank] = lrow;
            plan.order[rank] = i;
            plan.slot2piv[i] = rank;
            prow[rank] = lrow;
        } else {
            plan.slot2piv[i] = -1;
        }
        if (i == v - 1) s_npiv = rank + mine[i];
    }
    __syncthreads();
    const int npiv = s_npiv;
    // early non-pivots: rows of [fnpr, fnpr+npiv) that are not pivots, ascending
    // late pivots: pivot rows >= fnpr+npiv, ascending                       (conflux_opt.cpp:131-147)
    for (int i = t; i < npiv; i += T) {
        const int r = fnpr + i;
        bool isp = false;
        for (int j = 0; j < npiv; ++j) isp = isp || (prow[j] == r);
        mine[i] = isp ? 0 : 1;  // reuse: 1 = early non-pivot candidate at offset i
    }
    __syncthreads();
    for (int i = t; i < npiv; i += T) {
        if (mine[i]) {
            int rank = 0;
            for (int j = 0; j < i; ++j) rank += mine[j];
            plan.early[rank] = fnpr + i;
        }
        const int pr = prow[i];
        if (pr >= fnpr + npiv) {
            int rank = 0;
            for (int j = 0; j < npiv; ++j) rank += (prow[j] >= fnpr + npiv && prow[j] < pr) ? 1 : 0;
            plan.late[rank] = pr;
        }
    }
    if (t == 0) {
        int ne = 0;
        for (int j = 0; j < npiv; ++j) ne += mine[j];
        s_nel = ne;
        plan.npiv[0] = npiv;
        plan.nel[0] = ne;
    }
    __syncthreads();
    // rowsrc: new row r takes old row rowsrc[r]   (conflux_opt.hpp:193-216)
    const int nel = s_nel;
    for (int i = t; i < nel; i += T) plan.rowsrc[plan.late[i]] = plan.early[i];
    for (int i = t; i < npiv; i += T) plan.rowsrc[fnpr + i] = prow[i];
}

// ---------------------------------------------------------------- push_pivots_up phases (row moves)
__device__ __forceinline__ void copy_row_seg(double* __restrict__ dst, const double* __restrict__ src, int len, int chunk,
                                             int nchunks) {
    // len even, both 16-byte aligned; chunk `chunk` of `nchunks`
    const int n2 = len >> 1;
    const int per = (n2 + nchunks - 1) / nchunks;
    const int b = chunk * per, e = min(n2, b + per);
    const double2* s2 = reinterpret_cast<const double2*>(src);
    double2* d2 = reinterpret_cast<double2*>(dst);
    for (int i = b + threadIdx.x; i < e; i += blockDim.x) d2[i] = s2[i];
}
__global__ void push_phase1_kernel(const double* __restrict__ A, int64_t lda, int ncols, int col_lo, MovePlan plan, int v,
                                   double* __restrict__ tmp, double* __restrict__ a01raw, int64_t ld01, int c0) {
    const int npiv = plan.npiv[0];
    const int y = blockIdx.y;
    if (y < v) {  // tmp[i] = A[cur_piv[i]]
        if (y >= npiv) return;
        const int src = plan.cur_piv[y];
        copy_row_seg(tmp + (int64_t)y * lda + col_lo, A + (int64_t)src * lda + col_lo, ncols - col_lo, blockIdx.x,
                     gridDim.x);
    } else if (a01raw != nullptr) {  // pivot rows in tournament order (zeros where the pivot lives elsewhere)
        const int slot = y - v;
        const int p = plan.slot2piv[slot];
        const int len = ncols - c0;
        double* dst = a01raw + (int64_t)slot * ld01;
        if (p >= 0) {
            copy_row_seg(dst, A + (int64_t)plan.cur_piv[p] * lda + c0, len, blockIdx.x, gridDim.x);
        } else {
            const int n2 = len >> 1;
            const int per = (n2 + gridDim.x - 1) / gridDim.x;
            const int b = blockIdx.x * per, e = min(n2, b + per);
            double2* d2 = reinterpret_cast<double2*>(dst);
            for (int i = b + threadIdx.x; i < e; i += blockDim.x) d2[i] = make_double2(0.0, 0.0);
        }
    }
}
__global__ void push_phase2_kernel(double* __restrict__ A, int64_t lda, int ncols, int col_lo, MovePlan plan) {
    if ((int)blockIdx.y >= plan.nel[0]) return;
    const int src = plan.early[blockIdx.y], dst = plan.late[blockIdx.y];
    copy_row_seg(A + (int64_t)dst * lda + col_lo, A + (int64_t)src * lda + col_lo, ncols - col_lo, blockIdx.x, gridDim.x);
}
__global__ void push_phase3_kernel(double* __restrict__ A, int64_t lda, int ncols, int col_lo, int fnpr, MovePlan plan,
                                   const double* __restrict__ tmp) {
    if ((int)blockIdx.y >= plan.npiv[0]) return;
    copy_row_seg(A + (int64_t)(fnpr + blockIdx.y) * lda + col_lo, tmp + (int64_t)blockIdx.y * lda + col_lo, ncols - col_lo,
                 blockIdx.x, gridDim.x);
}

__global__ void gri_gather_kernel(const int* __restrict__ gri, int* __restrict__ gri_tmp, const int* __restrict__ rowsrc,
                                  int fnpr, int Ml) {
    const int r = fnpr + blockIdx.x * blockDim.x + threadIdx.x;
    if (r < Ml) gri_tmp[r] = gri[rowsrc[r]];
}
__global__ void gri_commit_kernel(int* __restrict__ gri, const int* __restrict__ gri_tmp, int* __restrict__ igri, int fnpr,
                                  int Ml, int v, int Px) {
    const int r = fnpr + blockIdx.x * blockDim.x + threadIdx.x;
    if (r < Ml) {
        const int g = gri_tmp[r];
        gri[r] = g;
        igri[(g / (v * Px)) * v + g % v] = r;
    }
}
__global__ void compact_panel_kernel(const double* __restrict__ PT, int64_t ldp, double* __restrict__ PT2, int64_t ldp2,
                                     const int* __restrict__ rowsrc, int fnpr_old, const int* __restrict__ npiv, int Ml) {
    const int fnpr_new = fnpr_old + npiv[0];
    const int rp = blockIdx.x * blockDim.x + threadIdx.x;
    const int c = blockIdx.y;
    if (fnpr_new + rp < Ml) PT2[(int64_t)c * ldp2 + rp] = PT[(int64_t)c * ldp + (rowsrc[fnpr_new + rp] - fnpr_old)];
}
__global__ void store_u_rows_kernel(double* __restrict__ A, int64_t lda, int fnpr_old, MovePlan plan,
                                    const double* __restrict__ U, int64_t ldu, int c0, int ncols) {
    if ((int)blockIdx.y >= plan.npiv[0]) return;
    const int i = blockIdx.y;
    copy_row_seg(A + (int64_t)(fnpr_old + i) * lda + c0, U + (int64_t)plan.order[i] * ldu, ncols, blockIdx.x, gridDim.x);
}
__global__ void store_diag_kernel(double* __restrict__ A, int64_t lda, int fnpr_old, MovePlan plan,
                                  const double* __restrict__ A00, int loff, int v) {
    if ((int)blockIdx.y >= plan.npiv[0]) return;
    const int i = blockIdx.y;
    const double* src = A00 + (int64_t)plan.order[i] * v;
    double* dst = A + (int64_t)(fnpr_old + i) * lda + loff;
    for (int c = threadIdx.x; c < v; c += blockDim.x) dst[c] = src[c];
}

__global__ void fill_kernel(double* p, int64_t n, double val) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = val;
}
__global__ void iota_gri_kernel(int* gri, int* igri, int Ml, int v, int Px, int pi) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < Ml) {
        gri[i] = (i % v) + ((i / v) * Px + pi) * v;  // conflux_opt.hpp:430-440
        igri[i] = i;
    }
}
__global__ void pack_bcast_kernel(const double* A00, const int* tags, int v, double* buf) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < v * v) buf[i] = A00[i];
    if (i < v) buf[v * v + i] = (double)tags[i];
}
__global__ void unpack_bcast_kernel(const double* buf, int v, double* A00, double* A00T, int* gpivots) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e < v * v) {
        const int i = e / v, c = e % v;
        const double x = buf[e];
        A00[e] = x;
        A00T[c * v + i] = x;
    }
    if (e < v) gpivots[e] = (int)buf[v * v + e];
}
__global__ void record_pivots_kernel(const int* gpivots, int v, int* hist, int k) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < v) hist[(int64_t)k * v + i] = gpivots[i];
}

// ---------------------------------------------------------------- residual helpers (validation, not on the hot path)
// LT[k][m] = L[m][k] (unit lower of the packed factors F, row-major n x n), U[k][c] = upper part
__global__ void split_factors_kernel(const double* __restrict__ F, int64_t ldf, int n, double* __restrict__ LT,
                                     double* __restrict__ U) {
    __shared__ double tile[32][33];
    const int r0 = blockIdx.y * 32, c0 = blockIdx.x * 32;
    for (int dy = threadIdx.y; dy < 32; dy += blockDim.y) {
        const int r = r0 + dy, c = c0 + threadIdx.x;
        double x = 0.0;
        if (r < n && c < n) x = F[(int64_t)r * ldf + c];
        tile[dy][threadIdx.x] = x;
        if (r < n && c < n) U[(int64_t)r * n + c] = (c >= r) ? x : 0.0;
    }
    __syncthreads();
    for (int dy = threadIdx.y; dy < 32; dy += blockDim.y) {
        const int k = c0 + dy, m = r0 + threadIdx.x;  // LT[k][m] = L[m][k]
        if (k < n && m < n) LT[(int64_t)k * n + m] = (m > k) ? tile[threadIdx.x][dy] : (m == k ? 1.0 : 0.0);
    }
}
__global__ void gather_perm_rows_kernel(const double* __restrict__ A, int64_t lda, const int* __restrict__ perm, int n,
                                        double* __restrict__ out) {
    const int r = blockIdx.x;
    const double* src = A + (int64_t)perm[r] * lda;
    double* dst = out + (int64_t)r * n;
    for (int c = blockIdx.y * blockDim.x + threadIdx.x; c < n; c += gridDim.y * blockDim.x) dst[c] = src[c];
}
// sum of a block's values in a fixed order (warp shuffles, then the warps' sums by warp 0); the result is in thread 0
__device__ __forceinline__ double block_sum(double s) {
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    __shared__ double w[32];
    if ((threadIdx.x & 31) == 0) w[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x < 32) {
        s = threadIdx.x < (blockDim.x >> 5) ? w[threadIdx.x] : 0.0;
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    }
    return s;
}
// Two passes with a fixed grid, so the sum is rounded the same way on every call: each CTA writes its partial sum, then
// one CTA adds the partials in index order.  (One pass with an atomicAdd per CTA rounds in whatever order the CTAs
// finish, so two runs over the same data could differ in the last bit.)
__global__ void sumsq_partial_kernel(const double* __restrict__ X, int64_t count, double* __restrict__ partials) {
    double s = 0.0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x)
        s = fma(X[i], X[i], s);
    s = block_sum(s);
    if (threadIdx.x == 0) partials[blockIdx.x] = s;
}
__global__ void sumsq_final_kernel(const double* __restrict__ partials, int n, double* __restrict__ out) {
    double s = 0.0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) s += partials[i];
    s = block_sum(s);
    if (threadIdx.x == 0) *out += s;
}

inline int row_chunks(int len) {
    int c = (len / 2 + 2047) / 2048;  // ~16 KB of double2 per CTA-chunk
    return c < 1 ? 1 : (c > 64 ? 64 : c);
}
}  // namespace

#define POST_LAUNCH()                     \
    do {                                  \
        CFLX_CUDA(cudaGetLastError());    \
        return CFLX_OK;                   \
    } while (0)

int launch_extract_panel_T(const double* A, int64_t lda, int64_t row0, int64_t col0, int n, int v, double* PT,
                           int64_t ldp, cudaStream_t s) {
    if (n <= 0) return CFLX_OK;
    dim3 grid((n + 31) / 32, (v + 31) / 32), block(32, 8);
    extract_panel_T_kernel<<<grid, block, 0, s>>>(A, lda, row0, col0, n, v, PT, ldp);
    POST_LAUNCH();
}
int launch_store_panel_T(double* A, int64_t lda, int64_t row0, int64_t col0, int n, int v, const double* LT, int64_t ldp,
                         cudaStream_t s) {
    if (n <= 0) return CFLX_OK;
    dim3 grid((n + 31) / 32, (v + 31) / 32), block(32, 8);
    store_panel_T_kernel<<<grid, block, 0, s>>>(A, lda, row0, col0, n, v, LT, ldp);
    POST_LAUNCH();
}
int launch_gather_winners(const double* PT, int64_t ldp, const int* tags, int n_valid, const int* perm, int v,
                          double* out_vals, int64_t ldo, int* out_tags, int dst0, cudaStream_t s) {
    const int64_t tot = (int64_t)v * v;
    gather_winners_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, s>>>(PT, ldp, tags, n_valid, perm, v, out_vals, ldo,
                                                                        out_tags, dst0);
    POST_LAUNCH();
}
int launch_gather_a00(const double* W, int64_t ldw, const int* perm, int v, int nb, double* A00, double* A00T,
                      cudaStream_t s) {
    const int64_t tot = (int64_t)v * v;
    gather_a00_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, s>>>(W, ldw, perm, v, nb, A00, A00T);
    POST_LAUNCH();
}
int launch_plan_moves(const int* gpivots, int v, int Px, int pi, int fnpr, int Ml, const int* igri, MovePlan plan,
                      cudaStream_t s) {
    plan_moves_kernel<<<1, 256, 2 * v * sizeof(int), s>>>(gpivots, v, Px, pi, fnpr, Ml, igri, plan);
    POST_LAUNCH();
}
int launch_push_phase1(const double* A, int64_t lda, int ncols, int col_lo, MovePlan plan, int v, double* tmp,
                       double* a01raw, int64_t ld01, int c0, cudaStream_t s) {
    dim3 grid(row_chunks(ncols), a01raw ? 2 * v : v);
    push_phase1_kernel<<<grid, 256, 0, s>>>(A, lda, ncols, col_lo, plan, v, tmp, a01raw, ld01, c0);
    POST_LAUNCH();
}
int launch_push_phase2(double* A, int64_t lda, int ncols, int col_lo, MovePlan plan, int v, cudaStream_t s) {
    dim3 grid(row_chunks(ncols), v);
    push_phase2_kernel<<<grid, 256, 0, s>>>(A, lda, ncols, col_lo, plan);
    POST_LAUNCH();
}
int launch_push_phase3(double* A, int64_t lda, int ncols, int col_lo, int fnpr, MovePlan plan, int v, const double* tmp,
                       cudaStream_t s) {
    dim3 grid(row_chunks(ncols), v);
    push_phase3_kernel<<<grid, 256, 0, s>>>(A, lda, ncols, col_lo, fnpr, plan, tmp);
    POST_LAUNCH();
}
int launch_update_gri(int* gri, int* gri_tmp, int* igri, const int* rowsrc, int fnpr, int Ml, int v, int Px,
                      cudaStream_t s) {
    const int n = Ml - fnpr;
    if (n <= 0) return CFLX_OK;
    gri_gather_kernel<<<(n + 255) / 256, 256, 0, s>>>(gri, gri_tmp, rowsrc, fnpr, Ml);
    gri_commit_kernel<<<(n + 255) / 256, 256, 0, s>>>(gri, gri_tmp, igri, fnpr, Ml, v, Px);
    POST_LAUNCH();
}
int launch_compact_panel(const double* PT, int64_t ldp, double* PT2, int64_t ldp2, const int* rowsrc, int fnpr_old,
                         const int* npiv, int Ml, int v, cudaStream_t s) {
    const int n = Ml - fnpr_old;
    if (n <= 0) return CFLX_OK;
    dim3 grid((n + 255) / 256, v);
    compact_panel_kernel<<<grid, 256, 0, s>>>(PT, ldp, PT2, ldp2, rowsrc, fnpr_old, npiv, Ml);
    POST_LAUNCH();
}
int launch_store_u_rows(double* A, int64_t lda, int fnpr_old, MovePlan plan, const double* U, int64_t ldu, int c0,
                        int ncols, int v, cudaStream_t s) {
    if (ncols <= 0) return CFLX_OK;
    dim3 grid(row_chunks(ncols), v);
    store_u_rows_kernel<<<grid, 256, 0, s>>>(A, lda, fnpr_old, plan, U, ldu, c0, ncols);
    POST_LAUNCH();
}
int launch_store_diag(double* A, int64_t lda, int fnpr_old, MovePlan plan, const double* A00, int loff, int v,
                      cudaStream_t s) {
    dim3 grid(1, v);
    store_diag_kernel<<<grid, 128, 0, s>>>(A, lda, fnpr_old, plan, A00, loff, v);
    POST_LAUNCH();
}
int launch_split_factors(const double* F, int64_t ldf, int n, double* LT, double* U, cudaStream_t s) {
    dim3 grid((n + 31) / 32, (n + 31) / 32), block(32, 8);  // n <= 2M rows
    split_factors_kernel<<<grid, block, 0, s>>>(F, ldf, n, LT, U);
    POST_LAUNCH();
}
int launch_gather_perm_rows(const double* A, int64_t lda, const int* perm, int n, double* out, cudaStream_t s) {
    dim3 grid(n, std::max(1, std::min(32, n / 256)));
    gather_perm_rows_kernel<<<grid, 256, 0, s>>>(A, lda, perm, n, out);
    POST_LAUNCH();
}
int launch_sumsq(const double* X, int64_t count, double* out, double* partials, cudaStream_t s) {
    sumsq_partial_kernel<<<SUMSQ_PARTIALS, 256, 0, s>>>(X, count, partials);
    CFLX_CUDA(cudaGetLastError());
    return launch_sum_partials(partials, SUMSQ_PARTIALS, out, s);
}
int launch_sum_partials(const double* partials, int n, double* out, cudaStream_t s) {
    sumsq_final_kernel<<<1, 1024, 0, s>>>(partials, n, out);
    POST_LAUNCH();
}
int launch_fill(double* p, int64_t n, double val, cudaStream_t s) {
    if (n <= 0) return CFLX_OK;
    fill_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(p, n, val);
    POST_LAUNCH();
}
int launch_iota_gri(int* gri, int* igri, int Ml, int v, int Px, int pi, cudaStream_t s) {
    iota_gri_kernel<<<(Ml + 255) / 256, 256, 0, s>>>(gri, igri, Ml, v, Px, pi);
    POST_LAUNCH();
}
int launch_pack_bcast(const double* A00, const int* tags, int v, double* buf, cudaStream_t s) {
    pack_bcast_kernel<<<(v * v + 255) / 256, 256, 0, s>>>(A00, tags, v, buf);
    POST_LAUNCH();
}
int launch_unpack_bcast(const double* buf, int v, double* A00, double* A00T, int* gpivots, cudaStream_t s) {
    unpack_bcast_kernel<<<(v * v + 255) / 256, 256, 0, s>>>(buf, v, A00, A00T, gpivots);
    POST_LAUNCH();
}
int launch_record_pivots(const int* gpivots, int v, int* hist, int k, cudaStream_t s) {
    record_pivots_kernel<<<(v + 255) / 256, 256, 0, s>>>(gpivots, v, hist, k);
    POST_LAUNCH();
}

}  // namespace cflx
