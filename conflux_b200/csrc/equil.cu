// conflux_b200/csrc/equil.cu -- equilibration and the expert drivers' device passes (cflx_lu_equilibrate, cflx_lu_svx,
// cflx_chol_equilibrate, cflx_chol_svx): LAPACK's dgeequ + dlaqge, dpoequ + dlaqsy and dgesvx's reciprocal pivot growth
// on the GPU grid.
//
// Every pass reads layer 0's local share A (Ml x Nl, conflux layout: local (r, c) is global (L.row(r), L.col(c))) once;
// it is HBM-bound.  What the ranks combine are maxima (and, for the Cholesky diagonal,
// sums with exactly one non-zero contributor per element), which are exact whatever the order: each rank writes its
// partial into an M-vector with zeros where it holds nothing, and one all-reduce over the world (ncclMax, or ncclSum for
// the diagonal) makes the vector bit-identical on every rank.  Inside a share, maxima of non-negative doubles are taken
// with integer atomicMax on their bit patterns (the order of non-negative IEEE doubles is that of their bits), again
// exact and order-independent.  The host then takes minima and maxima of the identical vectors, so every rank takes the
// same decisions.  The scaling is applied in LAPACK's operation order: r_i a, c_j a, (c_j r_i) a and (s_j s_i) a.
#include <climits>
#include <cmath>

#include "lu_state.h"

namespace cflx {
namespace {

constexpr int EQ_COLS = 128;  // local columns per CTA (one per thread) of the column passes
constexpr int EQ_ROWS = 256;  // local rows per CTA of the column passes

__device__ __forceinline__ void max_bits(double* out, double x) {  // x >= 0
    atomicMax(reinterpret_cast<unsigned long long*>(out), (unsigned long long)__double_as_longlong(x));
}

// one warp per local row: rowmax[g] = max_c |A[r][c]|
__global__ void row_max_kernel(const double* __restrict__ A, Layout L, double* __restrict__ rowmax) {
    const int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (r >= L.Ml) return;
    const double* a = A + (int64_t)r * L.Nl;
    double m = 0.0;
    for (int c = lane; c < L.Nl; c += 32) m = fmax(m, fabs(a[c]));
    for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (lane == 0) rowmax[L.row(r)] = m;
}

// colmax[g] = max over this CTA's rows of |A[r][c]| r[gr]; combined over the CTAs by atomicMax on the bits
__global__ void __launch_bounds__(EQ_COLS) col_max_kernel(const double* __restrict__ A, Layout L,
                                                          const double* __restrict__ rs, double* __restrict__ colmax) {
    const int c = blockIdx.x * EQ_COLS + threadIdx.x, r0 = blockIdx.y * EQ_ROWS, r1 = min(r0 + EQ_ROWS, L.Ml);
    if (c >= L.Nl) return;
    double m = 0.0;
    for (int r = r0; r < r1; ++r) m = fmax(m, fabs(A[(int64_t)r * L.Nl + c]) * rs[L.row(r)]);
    max_bits(colmax + L.col(c), m);
}

// diag[g] = a_gg on the diagonal tiles this share holds (global tile index < Nt)
__global__ void diag_kernel(const double* __restrict__ A, Layout L, double* __restrict__ diag) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= L.M) return;
    const int t = g / L.v, e = g % L.v;
    if (t >= L.Nt || !L.holds_diag(t)) return;
    diag[g] = A[(int64_t)(L.diag_row(t) + e) * L.Nl + L.diag_col(t) + e];
}

// x = 1 / min(max(x, small), 1 / small) elementwise (dgeequ's reciprocal scales)
__global__ void recip_kernel(double* x, int n, double small, double big) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) x[i] = 1.0 / fmin(fmax(x[i], small), big);
}

// dlaqge: 'R' r_i a, 'C' c_j a, 'B' (c_j r_i) a; a thread per local column, the rows strided over gridDim.y
template <char EQ>
__global__ void apply_kernel(double* __restrict__ A, Layout L, const double* __restrict__ rs,
                             const double* __restrict__ cs) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= L.Nl) return;
    const double cj = EQ == 'R' ? 1.0 : cs[L.col(c)];
    for (int r = blockIdx.y; r < L.Ml; r += gridDim.y) {
        const int64_t o = (int64_t)r * L.Nl + c;
        if (EQ == 'R') A[o] = rs[L.row(r)] * A[o];
        if (EQ == 'C') A[o] = cj * A[o];
        if (EQ == 'B') A[o] = (cj * rs[L.row(r)]) * A[o];
    }
}

// dlaqsy (UPLO = 'L'): (s_j s_i) a on the real tiles' entries with global row >= global column; nothing else is read
__global__ void sym_apply_kernel(double* __restrict__ A, Layout L, const double* __restrict__ ss) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= L.Nl) return;
    const int gj = L.col(c);
    if (gj / L.v >= L.Nt) return;
    for (int r = blockIdx.y; r < L.Ml; r += gridDim.y) {
        const int gi = L.row(r);
        if (gi / L.v >= L.Nt || gi < gj) continue;
        const int64_t o = (int64_t)r * L.Nl + c;
        A[o] = (ss[gj] * ss[gi]) * A[o];
    }
}

// first zero on the diagonal of U: out = min(1 + g) over the global diagonal entries this share holds with F_gg == 0
__global__ void zero_pivot_kernel(const double* __restrict__ F, Layout L, int* out) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= L.M) return;
    const int t = g / L.v, e = g % L.v;
    if (!L.holds_diag(t)) return;
    if (F[(int64_t)(L.diag_row(t) + e) * L.Nl + L.diag_col(t) + e] == 0.0) atomicMin(out, g + 1);
}

// out[0] = max |triu(F)|, out[1] = max |A| over the global columns < ncols of this share
__global__ void __launch_bounds__(EQ_COLS) growth_kernel(const double* __restrict__ F, const double* __restrict__ A,
                                                         Layout L, int ncols, double* out) {
    __shared__ double sh[2][EQ_COLS];
    const int c = blockIdx.x * EQ_COLS + threadIdx.x, r0 = blockIdx.y * EQ_ROWS, r1 = min(r0 + EQ_ROWS, L.Ml);
    double mu = 0.0, ma = 0.0;
    if (c < L.Nl) {
        const int gc = L.col(c);
        if (gc < ncols) {
            for (int r = r0; r < r1; ++r) {
                const int64_t o = (int64_t)r * L.Nl + c;
                ma = fmax(ma, fabs(A[o]));
                if (L.row(r) <= gc) mu = fmax(mu, fabs(F[o]));
            }
        }
    }
    sh[0][threadIdx.x] = mu;
    sh[1][threadIdx.x] = ma;
    __syncthreads();
    for (int w = EQ_COLS / 2; w > 0; w >>= 1) {
        if (threadIdx.x < w) {
            sh[0][threadIdx.x] = fmax(sh[0][threadIdx.x], sh[0][threadIdx.x + w]);
            sh[1][threadIdx.x] = fmax(sh[1][threadIdx.x], sh[1][threadIdx.x + w]);
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        max_bits(out, sh[0][0]);
        max_bits(out + 1, sh[1][0]);
    }
}

__global__ void scale_rows_kernel(double* __restrict__ X, int64_t ld, int M, int n, const double* __restrict__ d) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (int64_t)M * n) return;
    const int i = (int)(e / n), j = (int)(e % n);
    X[i * ld + j] = d[i] * X[i * ld + j];
}

// dlamch('S') and dlamch('S') / dlamch('P') (LAPACK's SMLNUM of dgeequ and SMALL of dlaqge / dlaqsy)
const double SAFMIN = std::ldexp(1.0, -1022), LAQ_SMALL = std::ldexp(1.0, -1022) / std::ldexp(1.0, -52);
constexpr double THRESH = 0.1;

// *a and *b (when b is not null) hold at least n doubles each; *cap is their common capacity
int grow_pair(double** a, double** b, size_t* cap, size_t n) {
    if (*a && n <= *cap) return CFLX_OK;
    cudaFree(*a);
    *a = nullptr;
    if (b) {
        cudaFree(*b);
        *b = nullptr;
    }
    *cap = 0;
    CFLX_TRY(dmalloc(a, n));
    if (b) CFLX_TRY(dmalloc(b, n));
    *cap = n;
    return CFLX_OK;
}

constexpr unsigned MAX_GRID_Y = 65535;

// all-reduce of an M-vector over the world, then its host copy
int reduce_vec(cflx_comm* c, double* d, int n, ncclRedOp_t op, std::vector<double>& h) {
    cudaStream_t s = c->stream;
    if (c->world_size > 1) CFLX_NCCL(ncclAllReduce(d, d, (size_t)n, ncclDouble, op, c->world, s));
    h.resize(n);
    CFLX_CUDA(cudaMemcpyAsync(h.data(), d, sizeof(double) * n, cudaMemcpyDeviceToHost, s));
    CFLX_CUDA(cudaStreamSynchronize(s));
    return CFLX_OK;
}

int launch_recip(double* x, int n, cudaStream_t s) {
    recip_kernel<<<(n + 255) / 256, 256, 0, s>>>(x, n, SAFMIN, 1.0 / SAFMIN);
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}
}  // namespace

// ---------------------------------------------------------------- per-share launches
int equil_row_max(const double* A, const Layout& L, double* rowmax, cudaStream_t s) {
    CFLX_CUDA(cudaMemsetAsync(rowmax, 0, sizeof(double) * L.M, s));
    if (L.Ml > 0 && L.Nl > 0) row_max_kernel<<<(L.Ml + 7) / 8, 256, 0, s>>>(A, L, rowmax);
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}

int equil_col_max(const double* A, const Layout& L, const double* r, double* colmax, cudaStream_t s) {
    CFLX_CUDA(cudaMemsetAsync(colmax, 0, sizeof(double) * L.M, s));
    if (L.Ml > 0 && L.Nl > 0) {
        const dim3 grid((L.Nl + EQ_COLS - 1) / EQ_COLS, (L.Ml + EQ_ROWS - 1) / EQ_ROWS);
        col_max_kernel<<<grid, EQ_COLS, 0, s>>>(A, L, r, colmax);
    }
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}

int equil_diag(const double* A, const Layout& L, double* diag, cudaStream_t s) {
    CFLX_CUDA(cudaMemsetAsync(diag, 0, sizeof(double) * L.M, s));
    diag_kernel<<<(L.M + 255) / 256, 256, 0, s>>>(A, L, diag);
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}

int diag_grid(const Grid& g, const double* A, double* d) {
    cflx_comm* c = g.comm;
    if (g.pk == 0) CFLX_TRY(equil_diag(A, g, d, c->stream));
    else CFLX_CUDA(cudaMemsetAsync(d, 0, sizeof(double) * g.M, c->stream));
    if (c->world_size > 1) CFLX_NCCL(ncclAllReduce(d, d, (size_t)g.M, ncclDouble, ncclSum, c->world, c->stream));
    return CFLX_OK;
}

int equil_apply(double* A, const Layout& L, const double* r, const double* c, char equed, cudaStream_t s) {
    if (L.Ml <= 0 || L.Nl <= 0 || equed == 'N') return CFLX_OK;
    const dim3 grid((L.Nl + 255) / 256, std::min((unsigned)L.Ml, MAX_GRID_Y));
    if (equed == 'R') apply_kernel<'R'><<<grid, 256, 0, s>>>(A, L, r, c);
    else if (equed == 'C') apply_kernel<'C'><<<grid, 256, 0, s>>>(A, L, r, c);
    else apply_kernel<'B'><<<grid, 256, 0, s>>>(A, L, r, c);
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}

int equil_sym_apply(double* A, const Layout& L, const double* sc, cudaStream_t s) {
    if (L.Ml <= 0 || L.Nl <= 0) return CFLX_OK;
    sym_apply_kernel<<<dim3((L.Nl + 255) / 256, std::min((unsigned)L.Ml, MAX_GRID_Y)), 256, 0, s>>>(A, L, sc);
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}

int launch_scale_rows(double* X, int64_t ld, int M, int n, const double* d, cudaStream_t s) {
    const int64_t tot = (int64_t)M * n;
    if (tot <= 0) return CFLX_OK;
    scale_rows_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, s>>>(X, ld, M, n, d);
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}

// ---------------------------------------------------------------- state
void equil_free(EquilState* e) {
    for (double* p : {e->in.r, e->in.c, e->fac.r, e->fac.c, e->qr, e->qc, e->B, e->X, e->growth, e->det}) cudaFree(p);
    cudaFree(e->ival);
    *e = EquilState{};
}

int equil_record_set(EquilRecord* dst, char equed, double rowcnd, double colcnd, const double* r, const double* c, int n,
                     cudaStream_t s) {
    dst->equed = equed;
    dst->rowcnd = rowcnd;
    dst->colcnd = colcnd;
    if (equed == 'N') return CFLX_OK;
    CFLX_TRY(grow_pair(&dst->r, &dst->c, &dst->cap, (size_t)n));
    CFLX_CUDA(cudaMemcpyAsync(dst->r, r, sizeof(double) * n, cudaMemcpyDeviceToDevice, s));
    if (c) CFLX_CUDA(cudaMemcpyAsync(dst->c, c, sizeof(double) * n, cudaMemcpyDeviceToDevice, s));
    return CFLX_OK;
}

int equil_pass_on(EquilState* e, int M, bool next_is_plain, cudaStream_t s) {
    const EquilRecord& in = e->in;
    CFLX_TRY(equil_record_set(&e->fac, in.equed, in.rowcnd, in.colcnd, in.r, in.c, M, s));
    if (next_is_plain) CFLX_TRY(equil_record_set(&e->in, 'N', 1.0, 1.0, nullptr, nullptr, M, s));
    return CFLX_OK;
}

int equil_grow(EquilState* e, int M, int ldn) {
    return grow_pair(&e->B, &e->X, &e->cap, (size_t)M * ldn);
}

// ---------------------------------------------------------------- dgeequ + dlaqge
int geequ_grid(const Grid& g, EquilState* e, double* A, bool apply, double* r_out, double* c_out, double* rowcnd,
               double* colcnd, double* amax, char* equed, int* info) {
    cflx_comm* c = g.comm;
    cudaStream_t s = c->stream;
    const int M = g.M;
    const bool layer0 = g.pk == 0;
    CFLX_TRY(grow_pair(&e->qr, &e->qc, &e->qcap, (size_t)M));
    double *r = e->qr, *cs = e->qc;
    std::vector<double> h;
    *info = 0;
    *rowcnd = *colcnd = 0.0;
    *equed = 'N';
    auto minmax = [&](double* lo, double* hi) {
        *lo = 1.0 / SAFMIN;
        *hi = 0.0;
        for (double x : h) *hi = std::max(*hi, x), *lo = std::min(*lo, x);
    };
    auto first_zero = [&]() {
        for (int i = 0; i < M; ++i)
            if (h[i] == 0.0) return i + 1;
        return 0;
    };
    // row maxima, then r = reciprocals
    if (layer0) CFLX_TRY(equil_row_max(A, g, r, s));
    else CFLX_CUDA(cudaMemsetAsync(r, 0, sizeof(double) * M, s));
    CFLX_TRY(reduce_vec(c, r, M, ncclMax, h));
    double rcmin, rcmax;
    minmax(&rcmin, &rcmax);
    *amax = rcmax;
    if (rcmin == 0.0) {  // dgeequ returns the row maxima in r and no column scales
        *info = first_zero();
        if (r_out) std::copy(h.begin(), h.end(), r_out);
        if (c_out) std::fill(c_out, c_out + M, 0.0);
        return CFLX_OK;
    }
    CFLX_TRY(launch_recip(r, M, s));
    CFLX_CUDA(cudaMemcpyAsync(h.data(), r, sizeof(double) * M, cudaMemcpyDeviceToHost, s));
    CFLX_CUDA(cudaStreamSynchronize(s));
    if (r_out) std::copy(h.begin(), h.end(), r_out);
    *rowcnd = std::max(rcmin, SAFMIN) / std::min(rcmax, 1.0 / SAFMIN);
    // column maxima of |a| r, then c = reciprocals
    if (layer0) CFLX_TRY(equil_col_max(A, g, r, cs, s));
    else CFLX_CUDA(cudaMemsetAsync(cs, 0, sizeof(double) * M, s));
    CFLX_TRY(reduce_vec(c, cs, M, ncclMax, h));
    minmax(&rcmin, &rcmax);
    if (rcmin == 0.0) {
        *info = M + first_zero();
        if (c_out) std::copy(h.begin(), h.end(), c_out);
        return CFLX_OK;
    }
    CFLX_TRY(launch_recip(cs, M, s));
    CFLX_CUDA(cudaMemcpyAsync(h.data(), cs, sizeof(double) * M, cudaMemcpyDeviceToHost, s));
    CFLX_CUDA(cudaStreamSynchronize(s));
    if (c_out) std::copy(h.begin(), h.end(), c_out);
    *colcnd = std::max(rcmin, SAFMIN) / std::min(rcmax, 1.0 / SAFMIN);
    if (!apply) return CFLX_OK;
    // dlaqge's decision
    const double large = 1.0 / LAQ_SMALL;
    if (*rowcnd >= THRESH && *amax >= LAQ_SMALL && *amax <= large) *equed = *colcnd >= THRESH ? 'N' : 'C';
    else *equed = *colcnd >= THRESH ? 'R' : 'B';
    if (layer0) CFLX_TRY(equil_apply(A, g, r, cs, *equed, s));
    CFLX_CUDA(cudaStreamSynchronize(s));
    return CFLX_OK;
}

// ---------------------------------------------------------------- dpoequ + dlaqsy
int poequ_grid(const Grid& g, EquilState* e, double* A, bool apply, double* s_out, double* scond, double* amax,
               char* equed, int* info) {
    cflx_comm* c = g.comm;
    cudaStream_t s = c->stream;
    const int N = g.M;
    CFLX_TRY(grow_pair(&e->qr, &e->qc, &e->qcap, (size_t)N));
    double* sc = e->qr;
    std::vector<double> h;
    *info = 0;
    *scond = 0.0;
    *equed = 'N';
    CFLX_TRY(diag_grid(g, A, sc));
    h.resize(N);
    CFLX_CUDA(cudaMemcpyAsync(h.data(), sc, sizeof(double) * N, cudaMemcpyDeviceToHost, s));
    CFLX_CUDA(cudaStreamSynchronize(s));
    double smin = h[0], smax = h[0];
    for (int i = 1; i < N; ++i) smin = std::min(smin, h[i]), smax = std::max(smax, h[i]);
    *amax = smax;
    if (smin <= 0.0) {  // dpoequ returns the diagonal in s
        for (int i = 0; i < N && !*info; ++i)
            if (h[i] <= 0.0) *info = i + 1;
        if (s_out) std::copy(h.begin(), h.end(), s_out);
        return CFLX_OK;
    }
    for (double& x : h) x = 1.0 / std::sqrt(x);
    if (s_out) std::copy(h.begin(), h.end(), s_out);
    CFLX_CUDA(cudaMemcpyAsync(sc, h.data(), sizeof(double) * N, cudaMemcpyHostToDevice, s));
    *scond = std::sqrt(smin) / std::sqrt(smax);
    if (apply) {
        const double large = 1.0 / LAQ_SMALL;
        *equed = (*scond >= THRESH && smax >= LAQ_SMALL && smax <= large) ? 'N' : 'Y';
        if (*equed == 'Y' && g.pk == 0) CFLX_TRY(equil_sym_apply(A, g, sc, s));
    }
    CFLX_CUDA(cudaStreamSynchronize(s));
    return CFLX_OK;
}

// ---------------------------------------------------------------- reciprocal pivot growth
int equil_zero_pivot(const double* F, const Layout& L, int* zero_pivot, cudaStream_t s) {
    const int big = INT_MAX;
    CFLX_CUDA(cudaMemcpyAsync(zero_pivot, &big, sizeof(int), cudaMemcpyHostToDevice, s));
    zero_pivot_kernel<<<(L.M + 255) / 256, 256, 0, s>>>(F, L, zero_pivot);
    CFLX_CUDA(cudaGetLastError());
    CFLX_CUDA(cudaStreamSynchronize(s));  // `big` is a host temporary
    return CFLX_OK;
}

int equil_growth(const double* F, const double* A, const Layout& L, int ncols, double* out2, cudaStream_t s) {
    CFLX_CUDA(cudaMemsetAsync(out2, 0, 2 * sizeof(double), s));
    if (L.Ml > 0 && L.Nl > 0) {
        const dim3 grid((L.Nl + EQ_COLS - 1) / EQ_COLS, (L.Ml + EQ_ROWS - 1) / EQ_ROWS);
        growth_kernel<<<grid, EQ_COLS, 0, s>>>(F, A, L, ncols, out2);
    }
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}

int zero_pivot_grid(const Grid& g, EquilState* e, const double* F, int* info) {
    cflx_comm* c = g.comm;
    cudaStream_t s = c->stream;
    if (!e->ival) CFLX_TRY(dmalloc(&e->ival, 1));
    if (g.pk == 0) {
        CFLX_TRY(equil_zero_pivot(F, g, e->ival, s));
    } else {  // only layer 0 holds the factors: this rank offers no zero pivot
        const int big = INT_MAX;
        CFLX_CUDA(cudaMemcpyAsync(e->ival, &big, sizeof(int), cudaMemcpyHostToDevice, s));
        CFLX_CUDA(cudaStreamSynchronize(s));
    }
    if (c->world_size > 1) CFLX_NCCL(ncclAllReduce(e->ival, e->ival, 1, ncclInt, ncclMin, c->world, s));
    int first = 0;
    CFLX_CUDA(cudaMemcpyAsync(&first, e->ival, sizeof(int), cudaMemcpyDeviceToHost, s));
    CFLX_CUDA(cudaStreamSynchronize(s));
    *info = first == INT_MAX ? 0 : first;
    return CFLX_OK;
}

int pivot_growth_grid(const Grid& g, EquilState* e, const double* F, const double* A, double* rpvgrw, int* info) {
    cflx_comm* c = g.comm;
    cudaStream_t s = c->stream;
    if (!e->growth) CFLX_TRY(dmalloc(&e->growth, 2));
    CFLX_TRY(zero_pivot_grid(g, e, F, info));
    const int ncols = *info ? *info : g.M;
    if (g.pk == 0) CFLX_TRY(equil_growth(F, A, g, ncols, e->growth, s));
    else CFLX_CUDA(cudaMemsetAsync(e->growth, 0, 2 * sizeof(double), s));
    if (c->world_size > 1) CFLX_NCCL(ncclAllReduce(e->growth, e->growth, 2, ncclDouble, ncclMax, c->world, s));
    double h[2];
    CFLX_CUDA(cudaMemcpyAsync(h, e->growth, sizeof(h), cudaMemcpyDeviceToHost, s));
    CFLX_CUDA(cudaStreamSynchronize(s));
    *rpvgrw = h[0] == 0.0 ? 1.0 : h[1] / h[0];  // dgesvx: dlange('M', A) / dlantr('M', 'U', AF)
    return CFLX_OK;
}

// ---------------------------------------------------------------- the expert drivers' solve
// B is scaled on the device, solved and refined there, and X is unscaled before the download
int svx_tail(EquilState* e, RefineCache* rc, const RefineOp& op, int nrhs, const double* B, int ldb, double* X, int ldx,
             double* ferr, double* berr, const double* pre, const double* post, double cnd, double rcond, int* info) {
    cudaStream_t s = op.grid.comm->stream;
    const int M = op.grid.M, ldn = (int)round_up(nrhs, 8);
    CFLX_TRY(equil_grow(e, M, ldn));
    double *dB = e->B, *dX = e->X;
    CFLX_CUDA(cudaMemcpy2DAsync(dB, ldn * sizeof(double), B, (size_t)ldb * sizeof(double), nrhs * sizeof(double), M,
                                cudaMemcpyDefault, s));
    if (pre) CFLX_TRY(launch_scale_rows(dB, ldn, M, nrhs, pre, s));
    CFLX_TRY(op.solve(false, nrhs, dB, ldn, dX, ldn));
    CFLX_TRY(refine_run(rc, op, nrhs, dB, ldn, dX, ldn, ferr, berr));
    if (post) CFLX_TRY(launch_scale_rows(dX, ldn, M, nrhs, post, s));
    CFLX_CUDA(cudaMemcpy2DAsync(X, (size_t)ldx * sizeof(double), dX, ldn * sizeof(double), nrhs * sizeof(double), M,
                                cudaMemcpyDefault, s));
    CFLX_CUDA(cudaStreamSynchronize(s));
    if (ferr && post)
        for (int j = 0; j < nrhs; ++j) ferr[j] /= cnd;
    *info = rcond < std::ldexp(1.0, -53) ? M + 1 : 0;
    return CFLX_OK;
}

}  // namespace cflx
