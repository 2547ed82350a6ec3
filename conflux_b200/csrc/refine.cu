// conflux_b200/csrc/refine.cu -- iterative refinement with error bounds (cflx_lu_refine, cflx_chol_refine): LAPACK's
// dgerfs / dporfs on the GPU grid.
//
// The residual kernels read layer 0's local share A (Ml x Nl, conflux layout: local (r, c) is global
// (Layout::row(r), Layout::col(c))) once and produce two partial products at once:
// P = op(A) X and Q = |op(A)| |X|.  They are the narrow GEMMs of the solve (solve.cu) with a second accumulator set fed
// by fabs of the same A and B fragments:
//   NN:  P, Q by local row,    from X gathered by local column (the LU, A X);
//   TN:  P, Q by local column, from X gathered by local row, A read transposed in place (the LU, A^T X);
//   symmetric lower (the Cholesky input, only its lower triangle stored): an NN pass over the entries with global row
//        >= global column, and a TN pass over those with global row > global column, both over the real tiles (global
//        tile index < Kappa) only.  Entries outside are masked by selecting 0.0, never by multiplying, so NaN left above
//        the diagonal or beyond Kappa does not reach the result; a CTA narrows its k range to the entries it may use, so
//        tiles above the diagonal cost no bandwidth.
// The doubled accumulators take registers: BN = 32 columns per CTA at most (NN and TN), and the TN kernel loads A 16 k
// rows at a time at that width (DESIGN.md section 7d has the register counts).  No floating-point atomics: every call
// gives the same bits.
//
// The partials of every layer-0 rank are all-gathered over the world and every rank adds them in the same fixed order,
// so op(A) x and |op(A)| |x| -- and everything the host branches on -- are bit-identical on every rank by construction.
#include <cmath>
#include <cstring>

#include "lu_state.h"
#include "narrow.cuh"

namespace cflx {
namespace {

struct ResidArgs {
    int M, N, K;  // output rows, right-hand sides, reduction length (local indices)
    const double* A;
    int64_t lda;
    const double* B;  // [K x N], ldb
    int64_t ldb;
    double *P, *Q;  // [M x N], ldo
    int64_t ldo;
    int v, Kappa;          // tile size; tiles with a global index >= Kappa are never read (masked modes)
    int Pm, pm, Pk, pk;    // grid extent and position of the output index (m) and of the reduction index (k)
};

__device__ __forceinline__ int first_tile(int g, int p, int P) { return g <= p ? 0 : (g - p + P - 1) / P; }
// number of local indices l (position p of P) with Layout::global(l, P, p, v) <= G
__device__ __forceinline__ int count_le(int G, int P, int p, int v) {
    const int T = G / v;
    return T % P == p ? (T / P) * v + G % v + 1 : first_tile(T + 1, p, P) * v;
}

enum { MASK_NONE = 0, MASK_LOWER = 1 /* gm >= gk */, MASK_STRICT_UPPER_T = 2 /* gk > gm */ };

template <int NT>
__device__ __forceinline__ void store_pq(const ResidArgs& r, const double (&acc)[NT][4], const double (&abs_acc)[NT][4],
                                         int64_t row_a, int64_t row_b, int n0, int t4) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int64_t row = h ? row_b : row_a;
        if (row >= r.M) continue;
#pragma unroll
        for (int j = 0; j < NT; ++j) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int col = n0 + 8 * j + 2 * t4 + e;
                if (col < r.N) {
                    r.P[row * r.ldo + col] = acc[j][2 * h + e];
                    r.Q[row * r.ldo + col] = abs_acc[j][2 * h + e];
                }
            }
        }
    }
}

__device__ __forceinline__ void abs4(const double (&a)[4], double (&o)[4]) {
#pragma unroll
    for (int i = 0; i < 4; ++i) o[i] = fabs(a[i]);
}

// P = A Xg, Q = |A| |Xg| with A [M x K] row-major read in place: the NN narrow GEMM (solve.cu gemm_narrow_kernel) with a
// second accumulator set.  MASK_LOWER keeps the entries with gm >= gk of the real tiles; the CTA stops at the last
// k its rows may use.
template <int NT, int MASK>
__global__ void __launch_bounds__(NW * 32, 1) resid_nn_kernel(ResidArgs r) {
    constexpr int BN = NarrowCfg<NT>::BN, LDP = NarrowCfg<NT>::LDP, STEPS = KC / 16;
    extern __shared__ double2 sB[];  // [2][KC / 2][LDP]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g4 = lane >> 2, t4 = lane & 3;
    const int64_t row0 = (int64_t)blockIdx.x * BM + warp * 16 + g4;
    const int n0 = blockIdx.y * BN;
    int K = r.K;
    int gm0 = 0, gm1 = 0;
    bool live0 = true, live1 = true;
    if (MASK == MASK_LOWER) {
        const int rlo = blockIdx.x * BM, rhi = min(rlo + BM, r.M) - 1;
        const int glo = Layout::global(rlo, r.Pm, r.pm, r.v), ghi = Layout::global(rhi, r.Pm, r.pm, r.v);
        K = glo / r.v >= r.Kappa ? 0 : min(K, min(count_le(ghi, r.Pk, r.pk, r.v), first_tile(r.Kappa, r.pk, r.Pk) * r.v));
        K = min(r.K, (K + 3) & ~3);  // a lane's four k indices lie in one tile (v % 4 == 0)
        gm0 = Layout::global((int)row0, r.Pm, r.pm, r.v);
        gm1 = Layout::global((int)row0 + 8, r.Pm, r.pm, r.v);
        live0 = gm0 / r.v < r.Kappa;
        live1 = gm1 / r.v < r.Kappa;
    }
    const NarrowArgs g{r.M, r.N, K, r.A, r.lda, r.B, r.ldb, nullptr, 0, nullptr, 0, 1.0, 0.0};
    const bool ok0 = row0 < r.M && live0, ok1 = row0 + 8 < r.M && live1;
    const double* a0p = r.A + (ok0 ? row0 * r.lda : 0);
    const double* a1p = r.A + (ok1 ? (row0 + 8) * r.lda : 0);
    double acc[NT][4], abs_acc[NT][4];
#pragma unroll
    for (int j = 0; j < NT; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[j][e] = abs_acc[j][e] = 0.0;

    auto keep2 = [](double2 x, bool k0, bool k1) { return make_double2(k0 ? x.x : 0.0, k1 ? x.y : 0.0); };
    auto load_a = [&](double2 (&a)[STEPS][4], int kc) {
#pragma unroll
        for (int s = 0; s < STEPS; ++s) {
            const int k = kc + 16 * s + 4 * t4;
            const bool kin = k < K;
            const double2 z = make_double2(0.0, 0.0);
            a[s][0] = (ok0 && kin) ? __ldg(reinterpret_cast<const double2*>(a0p + k)) : z;
            a[s][1] = (ok0 && kin) ? __ldg(reinterpret_cast<const double2*>(a0p + k + 2)) : z;
            a[s][2] = (ok1 && kin) ? __ldg(reinterpret_cast<const double2*>(a1p + k)) : z;
            a[s][3] = (ok1 && kin) ? __ldg(reinterpret_cast<const double2*>(a1p + k + 2)) : z;
            if (MASK == MASK_LOWER) {
                const int gk = Layout::global(k, r.Pk, r.pk, r.v);
                a[s][0] = keep2(a[s][0], gk <= gm0, gk + 1 <= gm0);
                a[s][1] = keep2(a[s][1], gk + 2 <= gm0, gk + 3 <= gm0);
                a[s][2] = keep2(a[s][2], gk <= gm1, gk + 1 <= gm1);
                a[s][3] = keep2(a[s][3], gk + 2 <= gm1, gk + 3 <= gm1);
            }
        }
    };
    if (K > 0) stage_b<NT>(g, 0, n0, sB);
    for (int kc = 0, c = 0; kc < K; kc += KC, ++c) {
        double2 a[STEPS][4];
        load_a(a, kc);
        cp_async_wait_all();
        __syncthreads();
        if (kc + KC < K) stage_b<NT>(g, kc + KC, n0, sB + ((c + 1) & 1) * NarrowCfg<NT>::STAGE);
        const double2* sb = sB + (c & 1) * NarrowCfg<NT>::STAGE;
#pragma unroll
        for (int s = 0; s < STEPS; ++s) {
            if (kc + 16 * s < K) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const double af[4] = {a[s][h].x, a[s][2 + h].x, a[s][h].y, a[s][2 + h].y};
                    double afa[4];
                    abs4(af, afa);
                    const double2* b_k = sb + (8 * s + 2 * t4 + h) * LDP + g4;
#pragma unroll
                    for (int j = 0; j < NT; ++j) {
                        const double2 bb = b_k[8 * j];
                        const double bf[2] = {bb.x, bb.y}, bfa[2] = {fabs(bb.x), fabs(bb.y)};
                        dmma16x8x8(acc[j], af, bf);
                        dmma16x8x8(abs_acc[j], afa, bfa);
                    }
                }
            }
        }
    }
    store_pq<NT>(r, acc, abs_acc, row0, row0 + 8, n0, t4);
}

// P = AT^T Xg, Q = |AT|^T |Xg| with AT [K x M] row-major read in place: the TN narrow GEMM (solve.cu
// gemm_narrow_tn_kernel) with a second accumulator set.  MASK_STRICT_UPPER_T keeps the entries with gk > gm of the real
// tiles (the strictly lower triangle of the stored matrix read as its transpose); the CTA starts at the first k any of
// its outputs may use.
constexpr int BM_TN = 32 * NW;
template <int NT>
struct ResidTnCfg {
    static constexpr int KA = NT >= 2 ? 16 : 32;  // k rows of AT per register load
};

template <int NT, int MASK>
__global__ void __launch_bounds__(NW * 32, 1) resid_tn_kernel(ResidArgs r) {
    constexpr int LDP = NarrowCfg<NT>::LDP, KA = ResidTnCfg<NT>::KA, SUB = KA / 16;
    extern __shared__ double2 sB[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g4 = lane >> 2, t4 = lane & 3;
    const int64_t ma = (int64_t)blockIdx.x * BM_TN + warp * 32 + 2 * g4, mb = ma + 16;
    const int n0 = blockIdx.y * NarrowCfg<NT>::BN;
    int k_lo = 0, K = r.K, gma = 0, gmb = 0;
    bool live_a = true, live_b = true;
    if (MASK == MASK_STRICT_UPPER_T) {
        const int glo = Layout::global(blockIdx.x * BM_TN, r.Pm, r.pm, r.v);
        const int k_hi = min(r.K, first_tile(r.Kappa, r.pk, r.Pk) * r.v);
        k_lo = glo / r.v >= r.Kappa ? k_hi : min(k_hi, count_le(glo, r.Pk, r.pk, r.v));
        K = k_hi - k_lo;
        gma = Layout::global((int)ma, r.Pm, r.pm, r.v);  // ma even, v even: ma + 1 is gma + 1
        gmb = Layout::global((int)mb, r.Pm, r.pm, r.v);
        live_a = gma / r.v < r.Kappa;
        live_b = gmb / r.v < r.Kappa;
    }
    const double* A = r.A + (int64_t)k_lo * r.lda;
    const NarrowArgs g{r.M, r.N, K, A, r.lda, r.B + (int64_t)k_lo * r.ldb, r.ldb, nullptr, 0, nullptr, 0, 1.0, 0.0};
    double acc[2][NT][4], abs_acc[2][NT][4];
#pragma unroll
    for (int p = 0; p < 2; ++p)
#pragma unroll
        for (int j = 0; j < NT; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[p][j][e] = abs_acc[p][j][e] = 0.0;

    auto load_pair = [&](const double* row, int64_t m) -> double2 {
        if (m + 1 < r.M) return __ldg(reinterpret_cast<const double2*>(row + m));
        return make_double2(m < r.M ? __ldg(row + m) : 0.0, 0.0);
    };
    auto load_a = [&](double2 (&a)[SUB][8], int kk) {
#pragma unroll
        for (int s = 0; s < SUB; ++s) {
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int k = kk + 16 * s + 4 * t4 + i;
                const double2 z = make_double2(0.0, 0.0);
                double2 xa = k < K && live_a ? load_pair(A + (int64_t)k * r.lda, ma) : z;
                double2 xb = k < K && live_b ? load_pair(A + (int64_t)k * r.lda, mb) : z;
                if (MASK == MASK_STRICT_UPPER_T) {
                    const int gk = Layout::global(k_lo + k, r.Pk, r.pk, r.v);
                    xa = make_double2(gk > gma ? xa.x : 0.0, gk > gma + 1 ? xa.y : 0.0);
                    xb = make_double2(gk > gmb ? xb.x : 0.0, gk > gmb + 1 ? xb.y : 0.0);
                }
                a[s][2 * i] = xa;
                a[s][2 * i + 1] = xb;
            }
        }
    };
    if (K > 0) stage_b<NT>(g, 0, n0, sB);
    for (int kc = 0, c = 0; kc < K; kc += KC, ++c) {
        const double2* sb = sB + (c & 1) * NarrowCfg<NT>::STAGE;
#pragma unroll 1
        for (int ks = 0; ks < KC && kc + ks < K; ks += KA) {
            double2 a[SUB][8];
            load_a(a, kc + ks);
            if (ks == 0) {
                cp_async_wait_all();
                __syncthreads();
                if (kc + KC < K) stage_b<NT>(g, kc + KC, n0, sB + ((c + 1) & 1) * NarrowCfg<NT>::STAGE);
            }
#pragma unroll
            for (int s = 0; s < SUB; ++s) {
                if (kc + ks + 16 * s < K) {
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const double2 *k0 = a[s] + 4 * h, *k1 = a[s] + 4 * h + 2;
                        const double af0[4] = {k0[0].x, k0[1].x, k1[0].x, k1[1].x};
                        const double af1[4] = {k0[0].y, k0[1].y, k1[0].y, k1[1].y};
                        double afa0[4], afa1[4];
                        abs4(af0, afa0);
                        abs4(af1, afa1);
                        const double2* b_k = sb + ((ks >> 1) + 8 * s + 2 * t4 + h) * LDP + g4;
#pragma unroll
                        for (int j = 0; j < NT; ++j) {
                            const double2 bb = b_k[8 * j];
                            const double bf[2] = {bb.x, bb.y}, bfa[2] = {fabs(bb.x), fabs(bb.y)};
                            dmma16x8x8(acc[0][j], af0, bf);
                            dmma16x8x8(acc[1][j], af1, bf);
                            dmma16x8x8(abs_acc[0][j], afa0, bfa);
                            dmma16x8x8(abs_acc[1][j], afa1, bfa);
                        }
                    }
                }
            }
        }
    }
#pragma unroll
    for (int p = 0; p < 2; ++p) store_pq<NT>(r, acc[p], abs_acc[p], ma + p, mb + p, n0, t4);
}

template <int NT, int MASK>
int launch_nn(const ResidArgs& r, cudaStream_t s) {
    using C = NarrowCfg<NT>;
    static PerDeviceMax cfg;
    if (cfg.raise(C::SMEM))
        CFLX_CUDA(cudaFuncSetAttribute(resid_nn_kernel<NT, MASK>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM));
    dim3 grid((unsigned)((r.M + BM - 1) / BM), (unsigned)((r.N + C::BN - 1) / C::BN));
    resid_nn_kernel<NT, MASK><<<grid, NW * 32, C::SMEM, s>>>(r);
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}

template <int NT, int MASK>
int launch_tn(const ResidArgs& r, cudaStream_t s) {
    using C = NarrowCfg<NT>;
    static PerDeviceMax cfg;
    if (cfg.raise(C::SMEM))
        CFLX_CUDA(cudaFuncSetAttribute(resid_tn_kernel<NT, MASK>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM));
    dim3 grid((unsigned)((r.M + BM_TN - 1) / BM_TN), (unsigned)((r.N + C::BN - 1) / C::BN));
    resid_tn_kernel<NT, MASK><<<grid, NW * 32, C::SMEM, s>>>(r);
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}

template <int MASK>
int dispatch_nn(const ResidArgs& r, cudaStream_t s) {
    if (r.N <= 8) return launch_nn<1, MASK>(r, s);
    if (r.N <= 16) return launch_nn<2, MASK>(r, s);
    return launch_nn<4, MASK>(r, s);  // slabs of 32 columns, one per blockIdx.y
}
template <int MASK>
int dispatch_tn(const ResidArgs& r, cudaStream_t s) {
    if (r.N <= 8) return launch_tn<1, MASK>(r, s);
    if (r.N <= 16) return launch_tn<2, MASK>(r, s);
    return launch_tn<4, MASK>(r, s);
}

// ---------------------------------------------------------------- assembly and the per-column backward error
struct AssembleArgs {
    const double* all;  // the partials of every world rank, `chunk` doubles apart: rows of 2 ldn (P, then Q)
    int64_t chunk;
    int Ml, Nl, ldn, nrhs, M;
    bool nn, tn;           // which partials a rank holds: NN rows [0, Ml), then TN rows [nn ? Ml : 0, + Nl)
    int v, Px, Py, Pz;
    const double* B;       // [M x ldn]
    double *R, *ratio, *W;  // [M x ldn]: b - op(A) x, the backward-error ratio, dgerfs' w
    double safe1, safe2, nzeps;
};

// every rank adds the same partials in the same order: for global row g (tile T), the NN partials of the ranks
// (T % Px, pj, 0), pj ascending, then the TN partials of the ranks (pi, T % Py, 0), pi ascending
__global__ void assemble_kernel(AssembleArgs a) {
    const int g = blockIdx.x, c = threadIdx.x + blockIdx.y * blockDim.x;
    if (g >= a.M || c >= a.nrhs) return;
    const int T = g / a.v, e = g % a.v;
    const int64_t ld2 = 2 * (int64_t)a.ldn;
    double p = 0.0, q = 0.0;
    if (a.nn) {
        const int64_t row = (int64_t)(T / a.Px) * a.v + e;
        for (int pj = 0; pj < a.Py; ++pj) {
            const double* src = a.all + (int64_t)(((T % a.Px) * a.Py + pj) * a.Pz) * a.chunk + row * ld2;
            p += src[c];
            q += src[a.ldn + c];
        }
    }
    if (a.tn) {
        const int64_t row = (a.nn ? a.Ml : 0) + (int64_t)(T / a.Py) * a.v + e;
        for (int pi = 0; pi < a.Px; ++pi) {
            const double* src = a.all + (int64_t)((pi * a.Py + T % a.Py) * a.Pz) * a.chunk + row * ld2;
            p += src[c];
            q += src[a.ldn + c];
        }
    }
    const int64_t o = (int64_t)g * a.ldn + c;
    const double b = a.B[o], r = b - p, s = q + fabs(b);
    a.R[o] = r;
    // dgerfs: s_i > safe2 ? |r_i| / s_i : (|r_i| + safe1) / (s_i + safe1);  w_i = |r_i| + nz eps s_i (+ safe1)
    a.ratio[o] = s > a.safe2 ? fabs(r) / s : (fabs(r) + a.safe1) / (s + a.safe1);
    a.W[o] = s > a.safe2 ? fabs(r) + a.nzeps * s : fabs(r) + a.nzeps * s + a.safe1;
}

// berr[c] = max over the rows of ratio[:, c], by a fixed tree (NaN wins)
constexpr int MAXT = 256;
__global__ void __launch_bounds__(MAXT) column_max_kernel(const double* __restrict__ ratio, int M, int ldn,
                                                          double* __restrict__ berr) {
    __shared__ double sh[MAXT];
    const int c = blockIdx.x;
    auto mx = [](double a, double b) { return (b > a || b != b) ? b : a; };
    double m = 0.0;
    for (int g = threadIdx.x; g < M; g += MAXT) m = mx(m, ratio[(int64_t)g * ldn + c]);
    sh[threadIdx.x] = m;
    __syncthreads();
    for (int w = MAXT / 2; w > 0; w >>= 1) {
        if (threadIdx.x < w) sh[threadIdx.x] = mx(sh[threadIdx.x], sh[threadIdx.x + w]);
        __syncthreads();
    }
    if (threadIdx.x == 0) berr[c] = sh[0];
}

// out[:, c] = active[c] ? in[:, c] : 0;  and X[:, c] += D[:, c] where active (dgerfs' daxpy)
__global__ void select_cols_kernel(const double* __restrict__ in, const int* __restrict__ active, int M, int ldn,
                                   double* __restrict__ out) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (int64_t)M * ldn) return;
    out[e] = active[e % ldn] ? in[e] : 0.0;
}
__global__ void add_cols_kernel(double* __restrict__ X, const double* __restrict__ D, const int* __restrict__ active, int M,
                                int ldn) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (int64_t)M * ldn) return;
    if (active[e % ldn]) X[e] = X[e] + D[e];
}

int grow(double** p, size_t n, size_t* have) {
    if (*p && n <= *have) return CFLX_OK;
    cudaFree(*p);
    *p = nullptr;
    *have = 0;
    CFLX_TRY(dmalloc(p, n));
    *have = n;
    return CFLX_OK;
}
}  // namespace

int launch_residual(ResidMode mode, const double* A, const Layout& L, const double* Xc, const double* Xr, int64_t ldx,
                    int nrhs, double* P, double* Q, int64_t ldo, cudaStream_t s) {
    const int64_t lda = L.Nl;
    const int Ml = L.Ml, Nl = L.Nl, v = L.v;
    if (nrhs <= 0) return CFLX_OK;
    if ((lda & 1) || (reinterpret_cast<uintptr_t>(A) & 15) || (v & 3)) {
        set_last_error("residual: unsupported layout lda=%lld v=%d (need even lda, v %% 4 == 0, 16-byte aligned A)",
                       (long long)lda, v);
        return CFLX_ERR_UNSUPPORTED;
    }
    // NN: output by local row (grid row position), reduction over local columns; TN: the other way round
    const ResidArgs nn{Ml, nrhs, Nl, A, lda, Xc, ldx, P, Q, ldo, v, L.Nt, L.Px, L.pi, L.Py, L.pj};
    const ResidArgs tn{Nl, nrhs, Ml, A, lda, Xr, ldx, P, Q, ldo, v, L.Nt, L.Py, L.pj, L.Px, L.pi};
    if (mode == ResidMode::NN) return Ml > 0 ? dispatch_nn<MASK_NONE>(nn, s) : CFLX_OK;
    if (mode == ResidMode::TN) return Nl > 0 ? dispatch_tn<MASK_NONE>(tn, s) : CFLX_OK;
    if (Ml > 0) CFLX_TRY(dispatch_nn<MASK_LOWER>(nn, s));
    ResidArgs t2 = tn;
    t2.P = P + (int64_t)Ml * ldo;
    t2.Q = Q + (int64_t)Ml * ldo;
    return Nl > 0 ? dispatch_tn<MASK_STRICT_UPPER_T>(t2, s) : CFLX_OK;
}

// ---------------------------------------------------------------- LAPACK dlacn2 as a reverse-communication step
void Lacn2::start(int n_) {
    n = n_;
    x.assign(n, 1.0 / n);
    v.assign(n, 0.0);
    isgn.assign(n, 0);
    est = 0.0;
    jump = 1;
    kase = 1;
}

int Lacn2::step() {
    constexpr int ITMAX = 5;
    auto asum = [&](const std::vector<double>& a) {
        double s = 0.0;
        for (double e : a) s += std::fabs(e);
        return s;
    };
    auto idamax = [&]() {
        int j = 0;
        double m = std::fabs(x[0]);
        for (int i = 1; i < n; ++i)
            if (std::fabs(x[i]) > m) m = std::fabs(x[i]), j = i;
        return j;
    };
    auto signs = [&]() {
        for (int i = 0; i < n; ++i) {
            x[i] = x[i] >= 0.0 ? 1.0 : -1.0;
            isgn[i] = (int)x[i];
        }
    };
    auto final_stage = [&]() {  // x_i = (-1)^i (1 + i / (n - 1))
        double altsgn = 1.0;
        for (int i = 0; i < n; ++i) {
            x[i] = altsgn * (1.0 + (double)i / (double)(n - 1));
            altsgn = -altsgn;
        }
        jump = 5;
        return kase = 1;
    };
    auto main_loop = [&]() {  // x = e_j
        std::fill(x.begin(), x.end(), 0.0);
        x[j] = 1.0;
        jump = 3;
        return kase = 1;
    };
    switch (jump) {
        case 1:  // x = A x of x = 1/n
            if (n == 1) {
                v[0] = x[0];
                est = std::fabs(v[0]);
                return kase = 0;
            }
            est = asum(x);
            signs();
            jump = 2;
            return kase = 2;
        case 2:  // x = A^T x of the sign vector
            j = idamax();
            iter = 2;
            return main_loop();
        case 3: {  // x = A e_j
            v = x;
            const double estold = est;
            est = asum(v);
            bool repeated = true;
            for (int i = 0; i < n && repeated; ++i) repeated = (x[i] >= 0.0 ? 1 : -1) == isgn[i];
            if (repeated || est <= estold) return final_stage();  // converged, or cycling
            signs();
            jump = 4;
            return kase = 2;
        }
        case 4: {  // x = A^T x of the sign vector
            const int jlast = j;
            j = idamax();
            if (x[jlast] != std::fabs(x[j]) && iter < ITMAX) {
                ++iter;
                return main_loop();
            }
            return final_stage();
        }
        default: {  // 5: x = A x of the alternating vector
            const double temp = 2.0 * (asum(x) / (double)(3 * n));
            if (temp > est) {
                v = x;
                est = temp;
            }
            return kase = 0;
        }
    }
}

// ---------------------------------------------------------------- the refinement driver
void refine_cache_free(RefineCache* rc) {
    for (double* p : {rc->X, rc->B, rc->R, rc->D, rc->rhs, rc->ratio, rc->W, rc->Xc, rc->Xr, rc->part, rc->all, rc->berr})
        cudaFree(p);
    for (int* p : {rc->gl_rows, rc->gl_cols, rc->active}) cudaFree(p);
    *rc = RefineCache{};
}

int refine_run(RefineCache* rc, const RefineOp& op, int nrhs, const double* B, int ldb, double* X, int ldx, double* ferr,
               double* berr_out) {
    const Grid& G = op.grid;
    cflx_comm* c = G.comm;
    cudaStream_t s = c->stream;
    const int M = G.M, Ml = G.Ml, Nl = G.Nl, v = G.v;
    const int ldn = (int)round_up(nrhs, 8);
    const bool nn = op.mode != ResidMode::TN, tn = op.mode != ResidMode::NN, layer0 = G.pk == 0;
    // local column (by_col) or row -> global row of X (clamped into X: masked entries never use the value)
    auto make_map = [&](int** dst, int n, bool by_col) -> int {
        if (*dst || n <= 0) return CFLX_OK;
        std::vector<int> m(n);
        for (int l = 0; l < n; ++l) {
            const int g = by_col ? G.col(l) : G.row(l);
            m[l] = g < M ? g : 0;
        }
        return solve_set_rows(dst, m, s);
    };
    if (layer0 && nn) CFLX_TRY(make_map(&rc->gl_cols, Nl, true));
    if (layer0 && tn) CFLX_TRY(make_map(&rc->gl_rows, Ml, false));
    const int prow = (nn ? Ml : 0) + (tn ? Nl : 0);
    const size_t mat = (size_t)M * ldn, chunk = (size_t)prow * 2 * ldn;
    if (rc->cap_m < mat) {  // the M x ldn buffers, grown together
        const std::initializer_list<double**> bufs = {&rc->X, &rc->B, &rc->R, &rc->D, &rc->rhs, &rc->ratio, &rc->W};
        for (double** p : bufs) {
            cudaFree(*p);
            *p = nullptr;
        }
        rc->cap_m = 0;
        for (double** p : bufs) CFLX_TRY(dmalloc(p, mat));
        rc->cap_m = mat;
    }
    CFLX_TRY(grow(&rc->Xc, (size_t)Nl * ldn, &rc->cap_c));
    CFLX_TRY(grow(&rc->Xr, (size_t)Ml * ldn, &rc->cap_r));
    CFLX_TRY(grow(&rc->part, chunk, &rc->cap_part));
    if (c->world_size > 1) CFLX_TRY(grow(&rc->all, chunk * c->world_size, &rc->cap_all));
    CFLX_TRY(grow(&rc->berr, (size_t)ldn, &rc->cap_berr));
    if (!rc->active || rc->cap_active < (size_t)ldn) {
        cudaFree(rc->active);
        rc->active = nullptr;
        CFLX_TRY(dmalloc(&rc->active, (size_t)ldn));
        rc->cap_active = ldn;
    }
    CFLX_CUDA(cudaMemsetAsync(rc->X, 0, sizeof(double) * mat, s));
    CFLX_CUDA(cudaMemsetAsync(rc->B, 0, sizeof(double) * mat, s));
    CFLX_CUDA(cudaMemcpy2DAsync(rc->X, ldn * sizeof(double), X, (size_t)ldx * sizeof(double), nrhs * sizeof(double), M,
                                cudaMemcpyDefault, s));
    CFLX_CUDA(cudaMemcpy2DAsync(rc->B, ldn * sizeof(double), B, (size_t)ldb * sizeof(double), nrhs * sizeof(double), M,
                                cudaMemcpyDefault, s));

    const double eps = std::ldexp(1.0, -53), safmin = std::ldexp(1.0, -1022);
    const double nz = (double)M + 1.0, safe1 = nz * safmin, safe2 = safe1 / eps;
    const double* all = c->world_size > 1 ? rc->all : rc->part;
    const AssembleArgs aa{all, (int64_t)chunk, Ml, Nl, ldn, nrhs, M, nn, tn, v, G.Px, G.Py, G.Pz, rc->B, rc->R,
                          rc->ratio, rc->W, safe1, safe2, nz * eps};
    std::vector<double> berr(nrhs);
    // one residual pass: R = B - op(A) X, the ratios, W, and berr on the host
    auto pass = [&]() -> int {
        if (layer0) {
            if (nn) CFLX_TRY(launch_gather_rows(rc->X, ldn, rc->gl_cols, Nl, ldn, rc->Xc, s));
            if (tn) CFLX_TRY(launch_gather_rows(rc->X, ldn, rc->gl_rows, Ml, ldn, rc->Xr, s));
            CFLX_TRY(launch_residual(op.mode, op.A, G, rc->Xc, rc->Xr, ldn, nrhs, rc->part, rc->part + ldn,
                                     2 * (int64_t)ldn, s));
        }
        if (c->world_size > 1) CFLX_NCCL(ncclAllGather(rc->part, rc->all, chunk, ncclDouble, c->world, s));
        assemble_kernel<<<dim3((unsigned)M, (unsigned)((nrhs + 127) / 128)), 128, 0, s>>>(aa);
        column_max_kernel<<<nrhs, MAXT, 0, s>>>(rc->ratio, M, ldn, rc->berr);
        CFLX_CUDA(cudaGetLastError());
        CFLX_CUDA(cudaMemcpyAsync(berr.data(), rc->berr, sizeof(double) * nrhs, cudaMemcpyDeviceToHost, s));
        CFLX_CUDA(cudaStreamSynchronize(s));
        return CFLX_OK;
    };

    // dgerfs, every column in lockstep: iterate while berr > eps, berr <= lstres / 2 and count <= ITMAX
    constexpr int ITMAX = 5;
    std::vector<int> count(nrhs, 1), active(ldn, 0);
    std::vector<double> lstres(nrhs, 3.0), col_berr(nrhs, 0.0);
    std::vector<char> refining(nrhs, 1);
    const unsigned eblocks = (unsigned)((mat + 255) / 256);
    for (;;) {
        CFLX_TRY(pass());
        bool any = false;
        for (int j = 0; j < nrhs; ++j) {
            active[j] = 0;
            if (!refining[j]) continue;
            col_berr[j] = berr[j];
            if (berr[j] > eps && 2.0 * berr[j] <= lstres[j] && count[j] <= ITMAX) {
                active[j] = 1;
                lstres[j] = berr[j];
                ++count[j];
                any = true;
            } else {
                refining[j] = 0;
            }
        }
        if (!any) break;
        CFLX_CUDA(cudaMemcpyAsync(rc->active, active.data(), sizeof(int) * ldn, cudaMemcpyHostToDevice, s));
        select_cols_kernel<<<eblocks, 256, 0, s>>>(rc->R, rc->active, M, ldn, rc->rhs);
        CFLX_CUDA(cudaGetLastError());
        CFLX_TRY(op.solve(false, nrhs, rc->rhs, ldn, rc->D, ldn));  // synchronises: `active` may change after it
        add_cols_kernel<<<eblocks, 256, 0, s>>>(rc->X, rc->D, rc->active, M, ldn);
        CFLX_CUDA(cudaGetLastError());
    }
    std::vector<double> hX((size_t)M * ldn);
    CFLX_CUDA(cudaMemcpyAsync(hX.data(), rc->X, sizeof(double) * mat, cudaMemcpyDeviceToHost, s));
    CFLX_CUDA(cudaStreamSynchronize(s));

    if (ferr) {
        // ||inv(op A)| w|_inf by dlacn2 on diag(w) inv(op A)^T (kase 1) and inv(op A) diag(w) (kase 2), one estimator per
        // column, all in lockstep: a round issues one solve per kind over the columns that ask for it
        std::vector<double> w(mat);
        CFLX_CUDA(cudaMemcpyAsync(w.data(), rc->W, sizeof(double) * mat, cudaMemcpyDeviceToHost, s));
        CFLX_CUDA(cudaStreamSynchronize(s));
        std::vector<Lacn2> est(nrhs);
        for (int j = 0; j < nrhs; ++j) est[j].start(M);
        std::vector<double> in(mat), out(mat);
        auto solve_round = [&](bool transposed, bool want1, bool want2) -> int {
            bool any = false;
            std::fill(in.begin(), in.end(), 0.0);
            for (int j = 0; j < nrhs; ++j) {
                const int k = est[j].kase;
                if (!((k == 1 && want1) || (k == 2 && want2))) continue;
                any = true;
                for (int i = 0; i < M; ++i) in[(size_t)i * ldn + j] = k == 2 ? w[(size_t)i * ldn + j] * est[j].x[i] : est[j].x[i];
            }
            if (!any) return CFLX_OK;
            CFLX_TRY(op.solve(transposed, nrhs, in.data(), ldn, out.data(), ldn));
            for (int j = 0; j < nrhs; ++j) {
                const int k = est[j].kase;
                if (!((k == 1 && want1) || (k == 2 && want2))) continue;
                for (int i = 0; i < M; ++i) {
                    const double y = out[(size_t)i * ldn + j];
                    est[j].x[i] = k == 1 ? w[(size_t)i * ldn + j] * y : y;
                }
                est[j].pending = true;
            }
            return CFLX_OK;
        };
        for (;;) {
            bool any = false;
            for (int j = 0; j < nrhs; ++j) any |= est[j].kase != 0;
            if (!any) break;
            if (op.symmetric) {
                CFLX_TRY(solve_round(false, true, true));
            } else {
                CFLX_TRY(solve_round(true, true, false));
                CFLX_TRY(solve_round(false, false, true));
            }
            for (int j = 0; j < nrhs; ++j)
                if (est[j].pending) {
                    est[j].pending = false;
                    est[j].step();
                }
        }
        for (int j = 0; j < nrhs; ++j) {
            double xmax = 0.0;
            for (int i = 0; i < M; ++i) xmax = std::max(xmax, std::fabs(hX[(size_t)i * ldn + j]));
            ferr[j] = xmax != 0.0 ? est[j].est / xmax : est[j].est;
        }
    }
    CFLX_CUDA(cudaMemcpy2DAsync(X, (size_t)ldx * sizeof(double), rc->X, ldn * sizeof(double), nrhs * sizeof(double), M,
                                cudaMemcpyDefault, s));
    CFLX_CUDA(cudaStreamSynchronize(s));
    if (berr_out) std::copy(col_berr.begin(), col_berr.end(), berr_out);
    return CFLX_OK;
}

}  // namespace cflx
