// conflux_b200/csrc/inverse.cu -- the explicit inverse from the factors left on the device: cflx_lu_inverse (LAPACK
// dgetri) and cflx_chol_inverse (dpotri, UPLO = 'L'), by block solves with the identity on the sweep engine (solve.cu).
//
// The inverse is built block column by block column, nc columns [c0, c0 + nc) at a time (nc a whole number of tiles).
// Each block is one run of the engine's sweeps on a right-hand side of ldn = round_up(nc, 8) columns:
//   * the identity block is written on the device into W on the ranks that seed a solve, (pi, 0, 0):
//     W[r][j] = (global row of r == c0 + j), after X, W and Z are zeroed as solve_seed zeroes them.  The LU seeds the
//     identity row map (it solves P A, as its condition estimate does); the Cholesky its real rows;
//   * the tiles that are exactly zero are skipped.  With T0 = c0 / v, the rows above c0 of the block stay zero through a
//     lower solve, so the forward sweep (L Y = E) starts at tile T0.  The Cholesky's backward sweep (L^T X = Y) stops at
//     T0, and its updates cover the local columns T0 <= gj < t only: dpotri's lower triangle needs the rows >= c0 of the
//     block.  The LU's backward sweep (U Z = Y) runs in full.  The flops of the block updates are then LAPACK's,
//     4/3 M^3 (LU) and 2/3 M^3 (Cholesky), against 2 M^3 for both without the skipping;
//   * solve_finish's world all-reduce assembles the block, the same bits on every rank (one contributor per element);
//   * the scatter writes block column j into this rank's share.  LU: column q = c0 + j of inv(P A) = inv(A) P^T is
//     column perm[q] of inv(A) = inv(P A) P, as dgetri's final column interchanges put it; every local row of that
//     column.  Cholesky: global column c0 + j, on the real tiles on and below the diagonal only; one zero pass sets the
//     rest of the share.
// These are right-inverse column solves: A X - I is small in norm.  dgetri's bound is on the left residual X A - I.
#include <algorithm>

#include "lu_state.h"

namespace cflx {
namespace {

constexpr int INV_COLS = 128;   // block columns (or local columns) per CTA, one per thread
constexpr int INV_ROWS = 2048;  // most CTAs along the local rows; each strides over the rest

// W[r][j] = (L.row(r) == c0 + j && j < nc) for r < rows, j < ldn
__global__ void inverse_seed_kernel(double* __restrict__ W, int ldn, Layout L, int rows, int c0, int nc) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= ldn) return;
    for (int r = blockIdx.y; r < rows; r += gridDim.y) W[(int64_t)r * ldn + j] = (j < nc && L.row(r) == c0 + j) ? 1.0 : 0.0;
}

// block column j of X into the share's column of global column perm[c0 + j] (LU) or c0 + j (Cholesky, real tiles on and
// below the diagonal only)
template <InvKind K>
__global__ void inverse_scatter_kernel(const double* __restrict__ X, int ldx, int c0, int nc, const int* __restrict__ perm,
                                       Layout L, double* __restrict__ out) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= nc) return;
    const int gc = K == InvKind::LU ? perm[c0 + j] : c0 + j, tc = gc / L.v;
    if (tc % L.Py != L.pj) return;
    const int lc = (tc / L.Py) * L.v + gc % L.v;
    if (lc >= L.Nl) return;
    for (int r = blockIdx.y; r < L.Ml; r += gridDim.y) {
        const int gr = L.row(r);
        if (K == InvKind::Chol && (gr / L.v >= L.Nt || gr / L.v < tc)) continue;
        out[(int64_t)r * L.Nl + lc] = X[(int64_t)gr * ldx + j];
    }
}

// zero on the entries the Cholesky scatter never writes: tiles above the diagonal and tiles with a global index >= Nt
__global__ void inverse_zero_kernel(Layout L, double* __restrict__ out) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= L.Nl) return;
    const int tc = L.col(c) / L.v;
    for (int r = blockIdx.y; r < L.Ml; r += gridDim.y) {
        const int tr = L.row(r) / L.v;
        if (tr >= L.Nt || tc >= L.Nt || tr < tc) out[(int64_t)r * L.Nl + c] = 0.0;
    }
}

dim3 grid_of(int cols, int rows) {
    return dim3((unsigned)((cols + INV_COLS - 1) / INV_COLS), (unsigned)std::max(1, std::min(rows, INV_ROWS)));
}
}  // namespace

int inverse_block_cols(int M, int v) {
    const int tiles = std::max(1, (CFLX_INV_NC + v / 2) / v);  // the whole number of tiles nearest CFLX_INV_NC
    return std::min(tiles * v, M);
}

int launch_inverse_seed(double* W, int ldn, const Layout& L, int rows, int c0, int nc, cudaStream_t s) {
    if (rows <= 0 || ldn <= 0) return CFLX_OK;
    inverse_seed_kernel<<<grid_of(ldn, rows), INV_COLS, 0, s>>>(W, ldn, L, rows, c0, nc);
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}

int launch_inverse_scatter(InvKind kind, const double* X, int ldx, int c0, int nc, const int* perm, const Layout& L,
                           double* out, cudaStream_t s) {
    if (nc <= 0 || L.Ml <= 0 || L.Nl <= 0) return CFLX_OK;
    if (kind == InvKind::LU)
        inverse_scatter_kernel<InvKind::LU><<<grid_of(nc, L.Ml), INV_COLS, 0, s>>>(X, ldx, c0, nc, perm, L, out);
    else
        inverse_scatter_kernel<InvKind::Chol><<<grid_of(nc, L.Ml), INV_COLS, 0, s>>>(X, ldx, c0, nc, perm, L, out);
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}

int launch_inverse_zero(const Layout& L, double* out, cudaStream_t s) {
    if (L.Ml <= 0 || L.Nl <= 0) return CFLX_OK;
    inverse_zero_kernel<<<grid_of(L.Nl, L.Ml), INV_COLS, 0, s>>>(L, out);
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}

namespace {
// the block loop into dst (a device share, or null: this rank joins the collectives only)
int inverse_blocks(SolveCache* sc, const SolveFactor& f, InvKind kind, const int* perm, double* dst, int ldn, int ncb) {
    const Grid& g = f.g;
    cudaStream_t s = g.comm->stream;
    const bool lu = kind == InvKind::LU;
    for (int c0 = 0; c0 < g.M; c0 += ncb) {
        const int nc = std::min(ncb, g.M - c0), T0 = c0 / g.v;
        CFLX_TRY(solve_seed(sc, f, ldn, 0, nullptr, 0, SolveSeed{false, nullptr, 0, nullptr}));  // zero X, W, Z
        if (g.pk == 0 && g.pj == 0) CFLX_TRY(launch_inverse_seed(sc->W, ldn, g, f.rows, c0, nc, s));
        if (lu) {  // L Y = E from tile T0 keeping Y_t as the owner's W rows, then U Z = Y in full
            CFLX_TRY(solve_row_sweep(sc, f, ldn, true, sc->W, g.Px, true, T0));
            CFLX_TRY(solve_row_sweep(sc, f, ldn, false, sc->X, 1, false));
        } else if (g.pk == 0) {  // L Y = E from tile T0 keeping Y_t in Z, then L^T X = Y down to tile T0
            CFLX_TRY(solve_row_sweep(sc, f, ldn, true, sc->Z, g.Py, false, T0));
            CFLX_TRY(solve_col_sweep(sc, f, ldn, false, Tri::LowerT, sc->X, 1, false, T0));
        }
        CFLX_TRY(solve_finish(sc, f, ldn, nc, nullptr, 0));
        if (dst) CFLX_TRY(launch_inverse_scatter(kind, sc->X, ldn, c0, nc, perm, g, dst, s));
    }
    if (dst && !lu) CFLX_TRY(launch_inverse_zero(g, dst, s));
    return CFLX_OK;
}
}  // namespace

int inverse_run(SolveCache* sc, const SolveFactor& f, InvKind kind, const int* perm, double* Ainv) {
    const Grid& g = f.g;
    cudaStream_t s = g.comm->stream;
    const int ncb = inverse_block_cols(g.M, g.v), ldn = (int)round_up(ncb, 8);
    CFLX_TRY(solve_cache_grow(sc, f, ldn, kind == InvKind::LU || g.pk == 0, kind == InvKind::Chol));
    // device output is written in place; host output goes through one temporary share, copied out once
    double* dst = nullptr;
    DevBuf<> tmp;
    const size_t n = (size_t)g.Ml * g.Nl;
    if (Ainv) {
        cudaPointerAttributes at{};
        const bool dev = cudaPointerGetAttributes(&at, Ainv) == cudaSuccess &&
                         (at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged);
        cudaGetLastError();  // an unknown host pointer is not an error here
        if (dev) dst = Ainv;
        else CFLX_TRY(tmp.alloc(n * sizeof(double)));
        if (tmp.p) dst = tmp.as<double>();
    }
    CFLX_TRY(inverse_blocks(sc, f, kind, perm, dst, ldn, ncb));
    if (tmp.p && cudaMemcpyAsync(Ainv, tmp.p, n * sizeof(double), cudaMemcpyDefault, s) != cudaSuccess) {
        set_last_error("inverse: copy of the share to the host failed");
        return CFLX_ERR_CUDA;
    }
    if (cudaStreamSynchronize(s) != cudaSuccess) {
        set_last_error("inverse: %s", cudaGetErrorString(cudaGetLastError()));
        return CFLX_ERR_CUDA;
    }
    return CFLX_OK;
}

}  // namespace cflx
