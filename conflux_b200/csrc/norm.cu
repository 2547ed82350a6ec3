// conflux_b200/csrc/norm.cu -- ||A||_1 of the input a factorisation keeps on the device (cflx_lu_rcond, cflx_chol_rcond).
//
// One pass over layer 0's local share A (Ml x Nl, conflux layout: local (r, c) is global (L.row(r), L.col(c))) writes per-CTA partial sums of |a| by local column and, for a matrix stored as its lower
// triangle, by local row; a second kernel adds them in a fixed order into an M-vector of this rank's share of every
// global column sum; an all-reduce over the world adds the ranks' shares, and the host takes the maximum.  No
// floating-point atomics: every call, and every rank, gets the same bits.  Every sum is compensated (Neumaier), so a
// column sum is within a few units in the last place of the exact one whatever the order: a long column of small
// entries under a large diagonal would otherwise lose about n u of it.
//
// A stored as its lower triangle (the Cholesky input): only the real tiles (global tile index < Nt) on and below the
// diagonal are read, and of the diagonal tiles only their lower triangle.  Column j of the symmetric matrix is the sum
// of its lower part (rows i >= j) plus the sum of the strictly lower part of ROW j (a_ji = a_ij for i < j).
#include <cmath>

#include "lu_state.h"

namespace cflx {
namespace {

constexpr int NCOL = 128;  // local columns per CTA (one per thread)
constexpr int NROW = 256;  // local rows per CTA
constexpr int SUB = 32;    // rows per shared-memory stage of the row sums

// s + c += a (Neumaier's compensated summation: s + c is the running sum to about 2u)
__device__ __forceinline__ void acc(double& s, double& c, double a) {
    const double t = s + a;
    c += fabs(s) >= fabs(a) ? (s - t) + a : (a - t) + s;
    s = t;
}

// colp[blockIdx.y][c] = sum of |A[r][c]| over this CTA's rows (masked); SYM: rowp[blockIdx.x][r] = the strictly lower
// part of row r over this CTA's columns
template <bool SYM>
__global__ void __launch_bounds__(NCOL) abs_sums_kernel(const double* __restrict__ A, Layout L, double* __restrict__ colp,
                                                        double* __restrict__ rowp) {
    const int Ml = L.Ml, Nl = L.Nl, v = L.v, Nt = L.Nt, Px = L.Px, Py = L.Py, pi = L.pi, pj = L.pj;
    __shared__ double sh[SYM ? SUB : 1][NCOL + 1];
    const int c = blockIdx.x * NCOL + threadIdx.x, r0 = blockIdx.y * NROW, r1 = min(r0 + NROW, Ml);
    const bool cin = c < Nl;
    const int gj = cin ? (c / v) * Py + pj : 0, cc = cin ? c % v : 0;  // global tile column, column in the tile
    double s = 0.0, sc = 0.0;
    if (!SYM) {
        if (cin) {
#pragma unroll 8
            for (int r = r0; r < r1; ++r) acc(s, sc, fabs(A[(int64_t)r * Nl + c]));
        }
    } else {
        const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
        for (int rs = r0; rs < r1; rs += SUB) {
            for (int k = 0; k < SUB; ++k) {
                const int r = rs + k;
                const int gi = (r / v) * Px + pi, rr = r % v;
                const bool real = cin && r < r1 && gi < Nt && gj < Nt && (gi > gj || (gi == gj && rr >= cc));
                const double a = real ? fabs(A[(int64_t)r * Nl + c]) : 0.0;
                acc(s, sc, a);
                sh[k][threadIdx.x] = (real && !(gi == gj && rr == cc)) ? a : 0.0;  // strictly lower: the row sums
            }
            __syncthreads();
            for (int k = warp; k < SUB; k += NCOL / 32) {
                double t = 0.0, tc = 0.0;
#pragma unroll
                for (int q = 0; q < NCOL / 32; ++q) acc(t, tc, sh[k][lane + 32 * q]);
                for (int o = 16; o > 0; o >>= 1) {  // the same tree on every call: (t, tc) pairs added pairwise
                    const double u = __shfl_xor_sync(0xffffffffu, t, o), uc = __shfl_xor_sync(0xffffffffu, tc, o);
                    tc += uc;
                    acc(t, tc, u);
                }
                if (lane == 0 && rs + k < r1) rowp[(int64_t)blockIdx.x * Ml + rs + k] = t + tc;
            }
            __syncthreads();
        }
    }
    if (cin) colp[(int64_t)blockIdx.y * Nl + c] = s + sc;
}

// out[g] = this rank's share of the sum of |a| over global column g, from the partials in a fixed order
template <bool SYM>
__global__ void column_sums_kernel(const double* __restrict__ colp, int ncp, const double* __restrict__ rowp, int nrp,
                                   Layout L, double* __restrict__ out) {
    const int M = L.M, Ml = L.Ml, Nl = L.Nl, v = L.v, Px = L.Px, Py = L.Py, pi = L.pi, pj = L.pj;
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= M) return;
    const int gt = g / v, e = g % v;
    double s = 0.0, sc = 0.0;
    if (gt % Py == pj && (gt / Py) * v + e < Nl) {
        const int c = (gt / Py) * v + e;
        for (int p = 0; p < ncp; ++p) acc(s, sc, colp[(int64_t)p * Nl + c]);
    }
    if (SYM && gt % Px == pi && (gt / Px) * v + e < Ml) {
        const int r = (gt / Px) * v + e;
        for (int p = 0; p < nrp; ++p) acc(s, sc, rowp[(int64_t)p * Ml + r]);
    }
    out[g] = s + sc;
}
// out[g] = the sum of |a| over local row r (global row g) of this share: one warp per row, each lane a compensated sum
// over the columns lane, lane + 32, ..., then the same shuffle tree as the row sums above
__global__ void row_abs_sums_kernel(const double* __restrict__ A, Layout L, double* __restrict__ out) {
    const int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (r >= L.Ml) return;
    const double* a = A + (int64_t)r * L.Nl;
    double t = 0.0, tc = 0.0;
    for (int c = lane; c < L.Nl; c += 32) acc(t, tc, fabs(a[c]));
    for (int o = 16; o > 0; o >>= 1) {
        const double u = __shfl_xor_sync(0xffffffffu, t, o), uc = __shfl_xor_sync(0xffffffffu, tc, o);
        tc += uc;
        acc(t, tc, u);
    }
    if (lane == 0) out[L.row(r)] = t + tc;
}
}  // namespace

void norm1_partials(const Layout& L, int* ncp, int* nrp) {
    *ncp = (L.Ml + NROW - 1) / NROW;
    *nrp = (L.Nl + NCOL - 1) / NCOL;
}

int launch_norm1_share(const double* A, const Layout& L, bool lower_sym, double* colp, double* rowp, double* out,
                       cudaStream_t s) {
    int ncp = 0, nrp = 0;
    norm1_partials(L, &ncp, &nrp);
    const dim3 grid(nrp, ncp);
    const int fin = (L.M + 255) / 256;
    if (lower_sym) {
        abs_sums_kernel<true><<<grid, NCOL, 0, s>>>(A, L, colp, rowp);
        column_sums_kernel<true><<<fin, 256, 0, s>>>(colp, ncp, rowp, nrp, L, out);
    } else {
        abs_sums_kernel<false><<<grid, NCOL, 0, s>>>(A, L, colp, rowp);
        column_sums_kernel<false><<<fin, 256, 0, s>>>(colp, ncp, rowp, nrp, L, out);
    }
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}

int launch_norminf_share(const double* A, const Layout& L, double* out, cudaStream_t s) {
    if (L.Ml <= 0) return CFLX_OK;
    row_abs_sums_kernel<<<(L.Ml + 7) / 8, 256, 0, s>>>(A, L, out);
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}

int norminf_grid(const Grid& g, const double* A, double* anorm) {
    cflx_comm* c = g.comm;
    cudaStream_t s = c->stream;
    const int M = g.M;
    DevBuf<double> out;
    CFLX_TRY(out.alloc((size_t)M));
    std::vector<double> h(M);
    CFLX_CUDA(cudaMemsetAsync(out, 0, sizeof(double) * M, s));
    if (g.pk == 0) CFLX_TRY(launch_norminf_share(A, g, out, s));  // only layer 0 holds the input
    if (c->world_size > 1) CFLX_NCCL(ncclAllReduce(out, out, (size_t)M, ncclDouble, ncclSum, c->world, s));
    CFLX_CUDA(cudaMemcpyAsync(h.data(), out, sizeof(double) * M, cudaMemcpyDeviceToHost, s));
    CFLX_CUDA(cudaStreamSynchronize(s));
    double m = 0.0;
    for (double x : h) m = std::isnan(x) ? x : std::max(m, x);  // dlange: a NaN row sum is the norm
    *anorm = m;
    return CFLX_OK;
}

int norm1_grid(const Grid& g, const double* A, bool lower_sym, double* anorm) {
    cflx_comm* c = g.comm;
    cudaStream_t s = c->stream;
    const int M = g.M, Ml = g.Ml, Nl = g.Nl, pk = g.pk;
    int ncp = 0, nrp = 0;
    norm1_partials(g, &ncp, &nrp);
    DevBuf<double> colp, rowp, out;
    CFLX_TRY(out.alloc((size_t)M));
    if (pk == 0) CFLX_TRY(colp.alloc((size_t)ncp * Nl));
    if (pk == 0 && lower_sym) CFLX_TRY(rowp.alloc((size_t)nrp * Ml));
    std::vector<double> h(M);
    if (pk != 0) {  // only layer 0 holds the input
        CFLX_CUDA(cudaMemsetAsync(out, 0, sizeof(double) * M, s));
    } else {
        CFLX_TRY(launch_norm1_share(A, g, lower_sym, colp, rowp, out, s));
    }
    if (c->world_size > 1) CFLX_NCCL(ncclAllReduce(out, out, (size_t)M, ncclDouble, ncclSum, c->world, s));
    CFLX_CUDA(cudaMemcpyAsync(h.data(), out, sizeof(double) * M, cudaMemcpyDeviceToHost, s));
    CFLX_CUDA(cudaStreamSynchronize(s));
    double m = 0.0;
    for (double x : h) m = std::isnan(x) ? x : std::max(m, x);  // dlange: a NaN column sum is the norm
    *anorm = m;
    return CFLX_OK;
}

}  // namespace cflx
