// conflux_b200/csrc/equil.cu -- equilibration and the expert drivers' device passes (cflx_lu_equilibrate[_b],
// cflx_lu_svx[x], cflx_chol_equilibrate[_b], cflx_chol_svx[x]): LAPACK's dgeequ / dgeequb + dlaqge, dpoequ / dpoequb +
// dlaqsy, and the reciprocal pivot growth of dgesvx and of dgesvxx / dposvxx (dla_gerpvgrw / dla_porpvgrw) on the GPU
// grid.
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

// amax[g] = max |a_ig|, fmx[g] = max |f_ig| over this CTA's rows of global column g < ncols, combined over the CTAs by
// atomicMax on the bits.  LU (SYM false): every row of A, the rows i <= g of F (U).  Cholesky (SYM): the real tiles'
// entries with g <= i < ncols of both.  Nothing outside the mask is read.
template <bool SYM>
__global__ void __launch_bounds__(EQ_COLS) growth_cols_kernel(const double* __restrict__ F, const double* __restrict__ A,
                                                              Layout L, int ncols, double* __restrict__ amax,
                                                              double* __restrict__ fmx) {
    const int c = blockIdx.x * EQ_COLS + threadIdx.x, r0 = blockIdx.y * EQ_ROWS, r1 = min(r0 + EQ_ROWS, L.Ml);
    if (c >= L.Nl) return;
    const int gc = L.col(c);
    if (gc >= ncols || (SYM && gc / L.v >= L.Nt)) return;
    double ma = 0.0, mf = 0.0;
#pragma unroll 4
    for (int r = r0; r < r1; ++r) {
        const int gr = L.row(r);
        const int64_t o = (int64_t)r * L.Nl + c;
        if (SYM) {
            if (gr >= gc && gr < ncols && gr / L.v < L.Nt) {
                ma = fmax(ma, fabs(A[o]));
                mf = fmax(mf, fabs(F[o]));
            }
        } else {
            ma = fmax(ma, fabs(A[o]));
            if (gr <= gc) mf = fmax(mf, fabs(F[o]));
        }
    }
    max_bits(amax + gc, ma);
    max_bits(fmx + gc, mf);
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

// RADIX**n of dgeequb / dpoequb for RADIX = 2, as an integer power evaluates it: 2^n, or 1 / 2^-n for n < 0 (0 once 2^-n
// overflows)
double pow2i(int n) { return n >= 0 ? std::ldexp(1.0, n) : 1.0 / std::ldexp(1.0, -n); }
// dgeequb's rounding of a positive maximum x to RADIX**INT(LOG(x) / LOGRDX).  The exponent comes from the host's log,
// the libm LAPACK calls: at an exact power of two it depends on how log rounds.
double round_pow2(double x) { return x > 0.0 ? pow2i((int)(std::log(x) / std::log(2.0))) : x; }

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
int equil_record_set(EquilRecord* dst, char equed, double rowcnd, double colcnd, const double* r, const double* c, int n,
                     cudaStream_t s) {
    dst->equed = equed;
    dst->rowcnd = rowcnd;
    dst->colcnd = colcnd;
    if (equed == 'N') return CFLX_OK;
    CFLX_TRY(grow_together({&dst->r, &dst->c}, (size_t)n));
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
    return grow_together({&e->B, &e->X}, (size_t)M * ldn);
}

// ---------------------------------------------------------------- dgeequ / dgeequb + dlaqge
int geequ_grid(const Grid& g, EquilState* e, double* A, bool apply, bool pow2, double* r_out, double* c_out,
               double* rowcnd, double* colcnd, double* amax, char* equed, int* info) {
    cflx_comm* c = g.comm;
    cudaStream_t s = c->stream;
    const int M = g.M;
    const bool layer0 = g.pk == 0;
    CFLX_TRY(grow_together({&e->qr, &e->qc}, (size_t)M));
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
    // dgeequb: the maxima rounded to powers of two on the host (h and its device copy d), before anything reads them
    auto rounded = [&](double* d) -> int {
        if (!pow2) return CFLX_OK;
        for (double& x : h) x = round_pow2(x);
        CFLX_CUDA(cudaMemcpyAsync(d, h.data(), sizeof(double) * M, cudaMemcpyHostToDevice, s));
        return CFLX_OK;
    };
    // row maxima, then r = reciprocals
    if (layer0) CFLX_TRY(equil_row_max(A, g, r, s));
    else CFLX_CUDA(cudaMemsetAsync(r, 0, sizeof(double) * M, s));
    CFLX_TRY(reduce_vec(c, r, M, ncclMax, h));
    CFLX_TRY(rounded(r));
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
    CFLX_TRY(rounded(cs));
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

// ---------------------------------------------------------------- dpoequ / dpoequb + dlaqsy
int poequ_grid(const Grid& g, EquilState* e, double* A, bool apply, bool pow2, double* s_out, double* scond,
               double* amax, char* equed, int* info) {
    cflx_comm* c = g.comm;
    cudaStream_t s = c->stream;
    const int N = g.M;
    CFLX_TRY(grow_together({&e->qr, &e->qc}, (size_t)N));
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
    const double tmp = -0.5 / std::log(2.0);  // dpoequb: RADIX**INT(TMP * LOG(a_ii)), the log on the host as in geequ_grid
    for (double& x : h) x = pow2 ? pow2i((int)(tmp * std::log(x))) : 1.0 / std::sqrt(x);
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

int equil_growth_cols(const double* F, const double* A, const Layout& L, bool sym, int ncols, double* out,
                      cudaStream_t s) {
    CFLX_CUDA(cudaMemsetAsync(out, 0, 2 * sizeof(double) * L.M, s));
    if (L.Ml > 0 && L.Nl > 0) {
        const dim3 grid((L.Nl + EQ_COLS - 1) / EQ_COLS, (L.Ml + EQ_ROWS - 1) / EQ_ROWS);
        if (sym) growth_cols_kernel<true><<<grid, EQ_COLS, 0, s>>>(F, A, L, ncols, out, out + L.M);
        else growth_cols_kernel<false><<<grid, EQ_COLS, 0, s>>>(F, A, L, ncols, out, out + L.M);
    }
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}

int zero_pivot_grid(const Grid& g, EquilState* e, const double* F, int* info) {
    cflx_comm* c = g.comm;
    cudaStream_t s = c->stream;
    if (!e->ival) CFLX_TRY(e->ival.alloc(1));
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

int growth_cols_grid(const Grid& g, EquilState* e, bool sym, const double* F, const double* A, int ncols,
                     std::vector<double>& h) {
    cflx_comm* c = g.comm;
    const int M = g.M;
    CFLX_TRY(e->growth.grow(2 * (size_t)M));
    if (g.pk == 0) CFLX_TRY(equil_growth_cols(F, A, g, sym, ncols, e->growth, c->stream));
    else CFLX_CUDA(cudaMemsetAsync(e->growth, 0, 2 * sizeof(double) * M, c->stream));
    return reduce_vec(c, e->growth, 2 * M, ncclMax, h);
}

double rpvgrw_cols(const std::vector<double>& h, int M, int ncols) {
    double rpvgrw = 1.0;
    for (int j = 0; j < ncols; ++j)
        if (h[M + j] != 0.0) rpvgrw = std::min(h[j] / h[M + j], rpvgrw);
    return rpvgrw;
}

int pivot_growth_grid(const Grid& g, EquilState* e, const double* F, const double* A, bool per_column, double* rpvgrw,
                      int* info) {
    const int M = g.M;
    CFLX_TRY(zero_pivot_grid(g, e, F, info));
    const int ncols = *info ? *info : M;
    std::vector<double> h;
    CFLX_TRY(growth_cols_grid(g, e, false, F, A, ncols, h));
    if (per_column) {
        *rpvgrw = rpvgrw_cols(h, M, ncols);
        return CFLX_OK;
    }
    // dgesvx: dlange('M', A) / dlantr('M', 'U', AF), the maxima of the two vectors (exact)
    double am = 0.0, fm = 0.0;
    for (int j = 0; j < M; ++j) am = std::max(am, h[j]), fm = std::max(fm, h[M + j]);
    *rpvgrw = fm == 0.0 ? 1.0 : am / fm;
    return CFLX_OK;
}

// ---------------------------------------------------------------- the expert drivers' solve
int svx_tail(EquilState* e, const RefineOp& op, int nrhs, const double* B, int ldb, double* X, int ldx,
             const RowTransform& pre, const RowTransform& post, const SvxRefine& refine) {
    cudaStream_t s = op.grid.comm->stream;
    const int M = op.grid.M, ldn = (int)round_up(nrhs, 8);
    CFLX_TRY(equil_grow(e, M, ldn));
    double *dB = e->B, *dX = e->X;
    CFLX_CUDA(cudaMemcpy2DAsync(dB, ldn * sizeof(double), B, (size_t)ldb * sizeof(double), nrhs * sizeof(double), M,
                                cudaMemcpyDefault, s));
    if (pre) CFLX_TRY(pre(dB, ldn, nrhs));
    CFLX_TRY(op.solve(false, nrhs, dB, ldn, dX, ldn));
    CFLX_TRY(refine(dB, ldn, dX, ldn));
    if (post) CFLX_TRY(post(dX, ldn, nrhs));
    CFLX_CUDA(cudaMemcpy2DAsync(X, (size_t)ldx * sizeof(double), dX, ldn * sizeof(double), nrhs * sizeof(double), M,
                                cudaMemcpyDefault, s));
    CFLX_CUDA(cudaStreamSynchronize(s));
    return CFLX_OK;
}

// the diagonal scaling by d (null: none) as a row transform of an M-row array
static RowTransform scale_rows(const Grid& g, const double* d) {
    if (!d) return RowTransform();
    return [&g, d](double* X, int64_t ld, int n) { return launch_scale_rows(X, ld, g.M, n, d, g.comm->stream); };
}

int svx_run(EquilState* e, RefineCache* rc, const RefineOp& op, int nrhs, const double* B, int ldb, double* X, int ldx,
            double* ferr, double* berr, const double* pre, const double* post, double cnd, double rcond, int* info) {
    auto refine = [&](const double* dB, int ldb_, double* dX, int ldx_) {
        return refine_run(rc, op, nrhs, dB, ldb_, dX, ldx_, ferr, berr);
    };
    CFLX_TRY(svx_tail(e, op, nrhs, B, ldb, X, ldx, scale_rows(op.grid, pre), scale_rows(op.grid, post), refine));
    if (ferr && post)
        for (int j = 0; j < nrhs; ++j) ferr[j] /= cnd;
    *info = rcond < std::ldexp(1.0, -53) ? op.grid.M + 1 : 0;
    return CFLX_OK;
}

int svxx_run(EquilState* e, RefineCache* rc, const RefineOp& op, int nrhs, const double* B, int ldb, double* X, int ldx,
             const double* pre, const double* post, const double* d, double rcond, bool cwise, double* berr,
             double* err_norm, double* err_comp, int* info) {
    auto refine = [&](const double* dB, int ldb_, double* dX, int ldx_) {
        return refine_x_run(rc, op, nrhs, dB, ldb_, dX, ldx_, d, rcond, cwise, berr, err_norm, err_comp, info);
    };
    return svx_tail(e, op, nrhs, B, ldb, X, ldx, scale_rows(op.grid, pre), scale_rows(op.grid, post), refine);
}

}  // namespace cflx
