// conflux_b200/csrc/solve_local.cu -- cflx_lu_solve_local and cflx_chol_solve_local: A X = B with B and X distributed in
// the conflux layout (ScaLAPACK's pdgetrs / pdpotrs), on the sweep engine (solve.cu).
//
// B and X are M x nrhs matrices tiled v x v like A: global tile (I, J) on grid position (I % Px, J % Py) at local tile
// (I / Px, J / Py) of a row-major share of Ml x rhs_local_cols(nrhs, v, Py).  The columns are solved in blocks of
// w <= inverse_block_cols(M, v) columns [c0, c0 + w), each on a right-hand side of ldn = round_up(w, 8) columns:
//   * pack: every layer-0 rank writes its share's entries of the block into a zeroed M x ldn buffer by global row (the
//     Cholesky: the real rows only, global tile index < Kappa).  Local columns with a global index >= nrhs are not read;
//   * assemble: one world all-reduce of that buffer, summed as 64-bit integers.  Exactly one rank contributes each
//     element and every other contributes zero bits, so the sum is B's block bit for bit (-0.0 and NaN payloads
//     included, which a floating-point sum of -0.0 and +0.0 would not keep);
//   * solve: the block is a device B of the existing solves (lu_sweeps, chol_sweeps), so each block is computed exactly
//     as cflx_lu_solve, cflx_lu_solve_trans or cflx_chol_solve computes those columns alone;
//   * scatter: the solved block (identical on every rank after solve_finish's all-reduce) into X's share, every layer.
// Block j is packed before it is scattered, and the blocks' columns are disjoint, so X may be B itself.  Host shares go
// through one temporary device share: the rows and columns the call reads and writes are a prefix of each (local rows
// before the first tile >= Kappa, local columns before the first global column >= nrhs).
#include <algorithm>

#include "lu_state.h"

namespace cflx {
namespace {

constexpr int SL_COLS = 128;   // block columns per CTA, one per thread
constexpr int SL_ROWS = 2048;  // most CTAs along the local rows; each strides over the rest

// the local column of global column gc on this share's grid column, or -1
__device__ __forceinline__ int local_col(const Layout& L, int gc) {
    const int tc = gc / L.v;
    return tc % L.Py == L.pj ? (tc / L.Py) * L.v + gc % L.v : -1;
}

// Bk[L.row(r)][j] = B[r][local column of c0 + j] for r < rows, j < w
__global__ void solve_local_pack_kernel(const double* __restrict__ B, int64_t ldb, Layout L, int rows, int c0, int w,
                                        double* __restrict__ Bk, int ldn) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= w) return;
    const int lc = local_col(L, c0 + j);
    if (lc < 0) return;
    for (int r = blockIdx.y; r < rows; r += gridDim.y) Bk[(int64_t)L.row(r) * ldn + j] = B[(int64_t)r * ldb + lc];
}

// X[r][local column of c0 + j] = Xk[L.row(r)][j] for r < rows, j < w
__global__ void solve_local_scatter_kernel(const double* __restrict__ Xk, int ldn, Layout L, int rows, int c0, int w,
                                           double* __restrict__ X, int64_t ldx) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= w) return;
    const int lc = local_col(L, c0 + j);
    if (lc < 0) return;
    for (int r = blockIdx.y; r < rows; r += gridDim.y) X[(int64_t)r * ldx + lc] = Xk[(int64_t)L.row(r) * ldn + j];
}

dim3 grid_of(int cols, int rows) {
    return dim3((unsigned)((cols + SL_COLS - 1) / SL_COLS), (unsigned)std::max(1, std::min(rows, SL_ROWS)));
}

// the local columns of a share whose global column is < nrhs: a prefix, as the global column grows with the local one
int valid_cols(int nrhs, int v, int Py, int pj) {
    int n = 0;
    for (int J = pj; J * v < nrhs; J += Py) n += std::min(v, nrhs - J * v);
    return n;
}

}  // namespace

int share_kind(const char* who, const Grid& g, const void* p, const char* what, bool* dev) {
    cudaPointerAttributes at{};
    *dev = cudaPointerGetAttributes(&at, p) == cudaSuccess &&
           (at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged);
    cudaGetLastError();  // an unknown host pointer is not an error here
    if (*dev && at.device != g.comm->device) {
        set_last_error("%s: %s is device memory of device %d, not this rank's device %d", who, what, at.device,
                       g.comm->device);
        return CFLX_ERR_ARG;
    }
    return CFLX_OK;
}

int rhs_local_cols(int nrhs, int v, int Py) { return v * (((nrhs + v - 1) / v + Py - 1) / Py); }

int solve_local_rows(const Layout& L, bool chol) {
    return chol ? std::min(L.Ml, first_local_tile(L.Nt, L.pi, L.Px) * L.v) : L.Ml;
}

int launch_solve_local_pack(const double* B, int64_t ldb, const Layout& L, int rows, int c0, int w, double* Bk, int ldn,
                            cudaStream_t s) {
    CFLX_CUDA(cudaMemsetAsync(Bk, 0, sizeof(double) * L.M * ldn, s));
    if (!B || rows <= 0 || w <= 0) return CFLX_OK;
    solve_local_pack_kernel<<<grid_of(w, rows), SL_COLS, 0, s>>>(B, ldb, L, rows, c0, w, Bk, ldn);
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}

int launch_solve_local_scatter(const double* Xk, int ldn, const Layout& L, int rows, int c0, int w, double* X, int64_t ldx,
                               cudaStream_t s) {
    if (rows <= 0 || w <= 0) return CFLX_OK;
    solve_local_scatter_kernel<<<grid_of(w, rows), SL_COLS, 0, s>>>(Xk, ldn, L, rows, c0, w, X, ldx);
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}

int rhs_args(const char* who, int nrhs, const double* B, int ldb, const double* X, int ldx, bool x_required) {
    REFUSE_FOR(who, nrhs < 1);
    REFUSE_FOR(who, !B);
    REFUSE_FOR(who, ldb < nrhs);
    REFUSE_FOR(who, x_required && !X);
    REFUSE_FOR(who, X && ldx < nrhs);
    return CFLX_OK;
}

int solve_local_args(const char* who, const Grid& g, int nrhs, const double* B, int ldb, const double* X, int ldx,
                     SolveLocalArgs* a) {
    REFUSE_FOR(who, nrhs < 1);
    const int local_cols = rhs_local_cols(nrhs, g.v, g.Py);
    if (g.pk != 0) B = nullptr;  // read on layer 0 only
    REFUSE_FOR(who, g.pk == 0 && !B);
    REFUSE_FOR(who, g.pk == 0 && ldb < local_cols);
    REFUSE_FOR(who, X && ldx < local_cols);
    if (B && X == B && ldx != ldb) {
        set_last_error("%s: X_local == B_local needs ldx == ldb (%d != %d)", who, ldx, ldb);
        return CFLX_ERR_ARG;
    }
    *a = SolveLocalArgs{nrhs, B, ldb, false, const_cast<double*>(X), ldx, false};
    if (B) CFLX_TRY(share_kind(who, g, B, "B_local", &a->b_dev));
    if (X) CFLX_TRY(share_kind(who, g, X, "X_local", &a->x_dev));
    return CFLX_OK;
}

int solve_local_run(const Grid& g, int rows, const SolveLocalArgs& a, const BlockSolve& solve) {
    cudaStream_t s = g.comm->stream;
    const int ncl = rhs_local_cols(a.nrhs, g.v, g.Py), cols = valid_cols(a.nrhs, g.v, g.Py, g.pj);
    const bool copy = rows > 0 && cols > 0;
    // a host share goes through one temporary device share (ld ncl), which holds B and then receives X when both are host
    DevBuf<> tmp;
    if ((a.B && !a.b_dev) || (a.X && !a.x_dev)) CFLX_TRY(tmp.alloc(sizeof(double) * std::max<size_t>(1, (size_t)rows * ncl)));
    const double* src = a.B;
    int64_t lds = a.ldb;
    if (a.B && !a.b_dev) {
        if (copy)
            CFLX_CUDA(cudaMemcpy2DAsync(tmp.p, sizeof(double) * ncl, a.B, sizeof(double) * a.ldb, sizeof(double) * cols,
                                        rows, cudaMemcpyHostToDevice, s));
        src = tmp.as<double>();
        lds = ncl;
    }
    double* dst = a.X;
    int64_t ldd = a.ldx;
    if (a.X && !a.x_dev) {
        dst = tmp.as<double>();
        ldd = ncl;
    }
    const int nc = inverse_block_cols(g.M, g.v);
    DevBuf<> Bk;
    CFLX_TRY(Bk.alloc(sizeof(double) * g.M * round_up(std::min(nc, a.nrhs), 8)));
    for (int c0 = 0; c0 < a.nrhs; c0 += nc) {
        const int w = std::min(nc, a.nrhs - c0), ldn = (int)round_up(w, 8);
        CFLX_TRY(launch_solve_local_pack(src, lds, g, rows, c0, w, Bk.as<double>(), ldn, s));
        if (g.P > 1)
            CFLX_NCCL(ncclAllReduce(Bk.p, Bk.p, (size_t)g.M * ldn, ncclUint64, ncclSum, g.comm->world, s));
        const double* Xk = nullptr;
        CFLX_TRY(solve(w, Bk.as<double>(), ldn, &Xk));
        if (dst) CFLX_TRY(launch_solve_local_scatter(Xk, ldn, g, rows, c0, w, dst, ldd, s));
    }
    if (a.X && !a.x_dev && copy)
        CFLX_CUDA(cudaMemcpy2DAsync(a.X, sizeof(double) * a.ldx, tmp.p, sizeof(double) * ncl, sizeof(double) * cols, rows,
                                    cudaMemcpyDeviceToHost, s));
    if (cudaStreamSynchronize(s) != cudaSuccess) {
        set_last_error("distributed solve: %s", cudaGetErrorString(cudaGetLastError()));
        return CFLX_ERR_CUDA;
    }
    return CFLX_OK;
}

}  // namespace cflx

extern "C" int cflx_rhs_local_cols(int nrhs, int v, int Py, int* cols_out) {
    REFUSE_IF(nrhs < 1);
    REFUSE_IF(v < 1);
    REFUSE_IF(Py < 1);
    REFUSE_IF(!cols_out);
    *cols_out = cflx::rhs_local_cols(nrhs, v, Py);
    return CFLX_OK;
}
