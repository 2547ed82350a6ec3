// conflux_b200/csrc/det.cu -- the determinant from the factors left on the device: cflx_lu_det (det(P A) = det(U), the
// sign of P from its cycles) and cflx_chol_det (det(A) = prod(l_ii)^2), as an exact-range product that cannot overflow.
//
// The diagonal is gathered by the equilibration's diagonal pass (equil.cu diag_grid: one non-zero contributor per
// element, so the world sum is exact and the M-vector is bit-identical on every rank).  One CTA of DET_THREADS then forms
// the product in a fixed order, so every rank and every call gets the same bits; oracle/det_ref.py restates it:
//   * a value x is the pair (m, e) = frexp(|x|), |x| = m 2^e with m in [0.5, 1): exact, subnormals included;
//   * a (x) b: p = m_a m_b, correctly rounded and in [0.25, 1); (f, k) = frexp(p); the result is (f, e_a + e_b + k).
//     a (/) b: the same with m_a / m_b, in (0.5, 2);
//   * thread t folds d[t c, min(n, (t + 1) c)), c = ceil(n / DET_THREADS), left to right from (0.5, 1), skipping the
//     entries that are zero or not finite; then slot t (x)= slot t + w for w = DET_THREADS / 2 .. 1 (t < w).  Each
//     divisor vector is reduced the same way, alongside;
//   * square: D (x)= D and S_i (x)= S_i; the result is D (/) S1 (/) S2 for the divisors given;
//   * the same pass counts the negative entries of d and the divisors (none when squaring), the first zero of d (min
//     index), and the first entry that is not finite in d or is not finite and non-zero in a divisor.  The result is
//     (NaN, 0) when that entry comes before the first zero, else (0, 0) when there is a zero.
#include <cmath>

#include "lu_state.h"

namespace cflx {
namespace {

struct Pair {
    double m;
    long long e;
};

// frexp(|x|) by the bits, x finite and non-zero: a subnormal is scaled by 2^64 first (exact)
__device__ __forceinline__ Pair split(double x) {
    long long b = __double_as_longlong(fabs(x)), bias = 1022;
    if ((b >> 52) == 0) {
        b = __double_as_longlong(__dmul_rn(fabs(x), 18446744073709551616.0));
        bias += 64;
    }
    return Pair{__longlong_as_double((b & 0x000fffffffffffffLL) | (1022LL << 52)), (b >> 52) - bias};
}

// (f, e + k) with (f, k) = frexp(p), p in [0.25, 2)
__device__ __forceinline__ Pair norm(double p, long long e) {
    if (p >= 1.0) return Pair{p * 0.5, e + 1};
    if (p < 0.5) return Pair{p * 2.0, e - 1};
    return Pair{p, e};
}

__device__ __forceinline__ Pair mul(Pair a, Pair b) { return norm(__dmul_rn(a.m, b.m), a.e + b.e); }
__device__ __forceinline__ Pair div(Pair a, Pair b) { return norm(__ddiv_rn(a.m, b.m), a.e - b.e); }

__device__ __forceinline__ bool finite(double x) { return fabs(x) <= 1.7976931348623157e308; }

// one slot of the tree: the partial products of d and of the divisors, the negative count, the first zero and the first
// bad entry (n when there is none)
struct Slot {
    Pair p[3];
    int neg, zero, bad;
};

__global__ void __launch_bounds__(DET_THREADS) det_kernel(const double* __restrict__ d, const double* __restrict__ s1,
                                                          const double* __restrict__ s2, int n, int square,
                                                          DetResult* out) {
    __shared__ Slot sh[DET_THREADS];
    const int t = threadIdx.x, c = (n + DET_THREADS - 1) / DET_THREADS;
    const double* v[3] = {d, s1, s2};
    Slot a{{{0.5, 1}, {0.5, 1}, {0.5, 1}}, 0, n, n};
    for (int i = t * c; i < min(n, (t + 1) * c); ++i) {
        for (int q = 0; q < 3; ++q) {
            if (!v[q]) continue;
            const double x = v[q][i];
            a.neg += x < 0.0;
            if (q == 0 && x == 0.0) a.zero = min(a.zero, i);
            else if (!finite(x) || x == 0.0) a.bad = min(a.bad, i);
            else a.p[q] = mul(a.p[q], split(x));
        }
    }
    sh[t] = a;
    __syncthreads();
    for (int w = DET_THREADS / 2; w > 0; w >>= 1) {
        if (t < w) {
            Slot& x = sh[t];
            const Slot& y = sh[t + w];
            for (int q = 0; q < 3; ++q) x.p[q] = mul(x.p[q], y.p[q]);
            x.neg += y.neg;
            x.zero = min(x.zero, y.zero);
            x.bad = min(x.bad, y.bad);
        }
        __syncthreads();
    }
    if (t) return;
    Slot r = sh[0];
    if (square)
        for (int q = 0; q < 3; ++q) r.p[q] = mul(r.p[q], r.p[q]);
    Pair p = r.p[0];
    if (s1) p = div(p, r.p[1]);
    if (s2) p = div(p, r.p[2]);
    out->neg = square ? 0 : (r.neg & 1);
    out->first_zero = r.zero < n ? r.zero + 1 : 0;
    out->nonfinite = r.bad < r.zero;
    if (out->nonfinite) p = Pair{__longlong_as_double(0x7ff8000000000000LL), 0};
    else if (r.zero < n) p = Pair{0.0, 0};
    out->mant = p.m;
    out->exp = p.e;
}
}  // namespace

int launch_det(const double* d, const double* s1, const double* s2, int n, bool square, DetResult* out,
               cudaStream_t s) {
    det_kernel<<<1, DET_THREADS, 0, s>>>(d, s1, s2, n, square ? 1 : 0, out);
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}

int det_grid(const Grid& g, EquilState* e, const double* F, bool square, const double* s1, const double* s2,
             DetResult* res) {
    cudaStream_t s = g.comm->stream;
    if (!e->det) CFLX_TRY(e->det.alloc((size_t)g.M + 4));  // the M-vector, then the DetResult
    DetResult* dr = reinterpret_cast<DetResult*>(e->det + g.M);
    CFLX_TRY(diag_grid(g, F, e->det));
    CFLX_TRY(launch_det(e->det, s1, s2, g.M, square, dr, s));
    CFLX_CUDA(cudaMemcpyAsync(res, dr, sizeof(DetResult), cudaMemcpyDeviceToHost, s));
    CFLX_CUDA(cudaStreamSynchronize(s));
    return CFLX_OK;
}

double det_log(const DetResult& r) {
    if (r.nonfinite) return std::nan("");
    if (r.first_zero) return -INFINITY;
    return std::log(r.mant) + (double)r.exp * 0.69314718055994530942;
}

}  // namespace cflx
