// conflux_b200/csrc/refine.cu -- iterative refinement with error bounds (cflx_lu_refine, cflx_chol_refine): LAPACK's
// dgerfs / dporfs on the GPU grid; and extra-precise refinement with trusted error bounds (cflx_lu_refine_x,
// cflx_chol_refine_x): dgerfsx / dporfsx, whose residuals come from the double-double kernels below (DESIGN.md §7h).
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

// ---------------------------------------------------------------- the double-double residual kernels (refine_x)
// Error-free transformations with the rounding spelled out (__dadd_rn / __dmul_rn are never contracted into an fma).
struct DD {
    double hi, lo;
};
__device__ __forceinline__ void two_sum(double a, double b, double& s, double& e) {
    s = __dadd_rn(a, b);
    const double bb = __dsub_rn(s, a);
    e = __dadd_rn(__dsub_rn(a, __dsub_rn(s, bb)), __dsub_rn(b, bb));
}
__device__ __forceinline__ DD dd_add(DD a, DD b) {
    double s, e;
    two_sum(a.hi, b.hi, s, e);
    e = __dadd_rn(e, __dadd_rn(a.lo, b.lo));
    DD r;
    two_sum(s, e, r.hi, r.lo);
    return r;
}
// Dot2 (Ogita, Rump, Oishi 2005) over the terms a (y + t): s collects the rounded products, c every rounding error
// (TwoProd by fma, TwoSum), and the tail's product, whose own rounding is second order
__device__ __forceinline__ void dot2_step(double a, double y, double t, double& s, double& c) {
    const double p = __dmul_rn(a, y), pe = fma(a, y, -p);
    double s2, q;
    two_sum(s, p, s2, q);
    s = s2;
    c = fma(a, t, __dadd_rn(c, __dadd_rn(q, pe)));
}

struct ResidXArgs {
    int M, N, K;  // output rows, right-hand sides, reduction length (local indices)
    const double* A;
    int64_t lda;
    const double *Y, *T;  // [K x N], ldb: the head and the tail of X gathered (T may be null: zero)
    int64_t ldb;
    double *Hi, *Lo;  // [M x N], ldo
    int64_t ldo;
    int v, Kappa, mask;
    int Pm, pm, Pk, pk;
};

__device__ __forceinline__ bool keep_entry(const ResidXArgs& r, int gm, int gk) {
    if (r.mask == MASK_NONE) return true;
    if (gm / r.v >= r.Kappa || gk / r.v >= r.Kappa) return false;
    return r.mask == MASK_LOWER ? gm >= gk : gk > gm;
}

constexpr int XW = 8;         // warps per CTA
constexpr int XROWS = 2;      // NN: output rows per warp
// NN: warp w of the CTA owns output rows blockIdx.x * XW * XROWS + w * XROWS + (0, 1); lane l reduces k = l, l + 32, ...
// (A read coalesced along its rows); the 32 lanes are combined by a butterfly of double-double additions.
template <int NB>
__global__ void __launch_bounds__(XW * 32) resid_x_nn_kernel(ResidXArgs r) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int m0 = (blockIdx.x * XW + warp) * XROWS, n0 = blockIdx.y * NB;
    double s[XROWS][NB], c[XROWS][NB];
    int gm[XROWS];
#pragma unroll
    for (int i = 0; i < XROWS; ++i) {
        gm[i] = Layout::global(m0 + i, r.Pm, r.pm, r.v);
#pragma unroll
        for (int j = 0; j < NB; ++j) s[i][j] = c[i][j] = 0.0;
    }
    for (int k = lane; k < r.K; k += 32) {
        const int gk = Layout::global(k, r.Pk, r.pk, r.v);
        double y[NB], t[NB];
#pragma unroll
        for (int j = 0; j < NB; ++j) {
            const bool in = n0 + j < r.N;
            y[j] = in ? r.Y[(int64_t)k * r.ldb + n0 + j] : 0.0;
            t[j] = in && r.T ? r.T[(int64_t)k * r.ldb + n0 + j] : 0.0;
        }
#pragma unroll
        for (int i = 0; i < XROWS; ++i) {
            if (m0 + i >= r.M) continue;
            const double raw = r.A[(int64_t)(m0 + i) * r.lda + k];
            const double a = keep_entry(r, gm[i], gk) ? raw : 0.0;  // selected away, never multiplied
#pragma unroll
            for (int j = 0; j < NB; ++j) dot2_step(a, y[j], t[j], s[i][j], c[i][j]);
        }
    }
#pragma unroll
    for (int i = 0; i < XROWS; ++i)
#pragma unroll
        for (int j = 0; j < NB; ++j) {
            DD p;
            two_sum(s[i][j], c[i][j], p.hi, p.lo);
#pragma unroll
            for (int w = 16; w > 0; w >>= 1) {
                const DD o{__shfl_xor_sync(0xffffffffu, p.hi, w), __shfl_xor_sync(0xffffffffu, p.lo, w)};
                p = lane & w ? dd_add(o, p) : dd_add(p, o);  // both lanes of a pair form the same sum
            }
            if (lane == 0 && m0 + i < r.M && n0 + j < r.N) {
                r.Hi[(int64_t)(m0 + i) * r.ldo + n0 + j] = p.hi;
                r.Lo[(int64_t)(m0 + i) * r.ldo + n0 + j] = p.lo;
            }
        }
}

// TN: lane l of every warp owns output m = blockIdx.x * 32 + l (A^T: column m of A, read coalesced along A's rows);
// warp w reduces k = w, w + XW, ...; the XW warps' partials are combined in shared memory by a fixed tree.
template <int NB>
__global__ void __launch_bounds__(XW * 32) resid_x_tn_kernel(ResidXArgs r) {
    __shared__ DD sh[XW][32][NB];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int m = blockIdx.x * 32 + lane, n0 = blockIdx.y * NB;
    const bool live = m < r.M;
    const int gm = Layout::global(live ? m : 0, r.Pm, r.pm, r.v);
    double s[NB], c[NB];
#pragma unroll
    for (int j = 0; j < NB; ++j) s[j] = c[j] = 0.0;
    for (int k = warp; k < r.K; k += XW) {
        const int gk = Layout::global(k, r.Pk, r.pk, r.v);
        const double raw = live ? r.A[(int64_t)k * r.lda + m] : 0.0;
        const double a = live && keep_entry(r, gm, gk) ? raw : 0.0;
#pragma unroll
        for (int j = 0; j < NB; ++j) {
            const bool in = n0 + j < r.N;
            const double y = in ? r.Y[(int64_t)k * r.ldb + n0 + j] : 0.0;
            const double t = in && r.T ? r.T[(int64_t)k * r.ldb + n0 + j] : 0.0;
            dot2_step(a, y, t, s[j], c[j]);
        }
    }
#pragma unroll
    for (int j = 0; j < NB; ++j) two_sum(s[j], c[j], sh[warp][lane][j].hi, sh[warp][lane][j].lo);
    __syncthreads();
    for (int w = XW / 2; w > 0; w >>= 1) {
        if (warp < w)
#pragma unroll
            for (int j = 0; j < NB; ++j) sh[warp][lane][j] = dd_add(sh[warp][lane][j], sh[warp + w][lane][j]);
        __syncthreads();
    }
    if (warp == 0 && live)
#pragma unroll
        for (int j = 0; j < NB; ++j)
            if (n0 + j < r.N) {
                r.Hi[(int64_t)m * r.ldo + n0 + j] = sh[0][lane][j].hi;
                r.Lo[(int64_t)m * r.ldo + n0 + j] = sh[0][lane][j].lo;
            }
}

template <int NB>
int launch_x(const ResidXArgs& r, bool tn, cudaStream_t s) {
    if (r.M <= 0) return CFLX_OK;
    const unsigned gy = (unsigned)((r.N + NB - 1) / NB);
    if (tn) resid_x_tn_kernel<NB><<<dim3((unsigned)((r.M + 31) / 32), gy), XW * 32, 0, s>>>(r);
    else resid_x_nn_kernel<NB><<<dim3((unsigned)((r.M + XW * XROWS - 1) / (XW * XROWS)), gy), XW * 32, 0, s>>>(r);
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}
int dispatch_x(const ResidXArgs& r, bool tn, cudaStream_t s) {
    if (r.N <= 1) return launch_x<1>(r, tn, s);
    if (r.N <= 2) return launch_x<2>(r, tn, s);
    if (r.N <= 4) return launch_x<4>(r, tn, s);
    return launch_x<8>(r, tn, s);  // slabs of 8 columns, one per blockIdx.y
}

// ---------------------------------------------------------------- assembly and the per-column backward error
// (AssembleArgs: lu_state.h)
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
    if (a.Q) a.Q[o] = q;
    if (a.lin_berr) {
        a.ratio[o] = s != 0.0 ? (fabs(r) + a.safe1) / s : 0.0;
        return;
    }
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

// refine_x: R = b - sum of the double-double partials (rows of 2 ldn: Hi, then Lo), added in assemble_kernel's order in
// double-double, b subtracted in double-double and rounded once
__global__ void assemble_x_kernel(AssembleArgs a) {
    const int g = blockIdx.x, c = threadIdx.x + blockIdx.y * blockDim.x;
    if (g >= a.M || c >= a.nrhs) return;
    const int T = g / a.v, e = g % a.v;
    const int64_t ld2 = 2 * (int64_t)a.ldn;
    DD p{0.0, 0.0};
    if (a.nn) {
        const int64_t row = (int64_t)(T / a.Px) * a.v + e;
        for (int pj = 0; pj < a.Py; ++pj) {
            const double* src = a.all + (int64_t)(((T % a.Px) * a.Py + pj) * a.Pz) * a.chunk + row * ld2;
            p = dd_add(p, DD{src[c], src[a.ldn + c]});
        }
    }
    if (a.tn) {
        const int64_t row = (a.nn ? a.Ml : 0) + (int64_t)(T / a.Py) * a.v + e;
        for (int pi = 0; pi < a.Px; ++pi) {
            const double* src = a.all + (int64_t)((pi * a.Py + T % a.Py) * a.Pz) * a.chunk + row * ld2;
            p = dd_add(p, DD{src[c], src[a.ldn + c]});
        }
    }
    const int64_t o = (int64_t)g * a.ldn + c;
    double s, err;
    two_sum(a.B[o], -p.hi, s, err);
    a.R[o] = __dadd_rn(s, __dsub_rn(err, p.lo));
}

// refine_x's per-column quantities of one round, by a fixed tree: {normy = max |y|, normx = max |y| d, normdx =
// max |dy| d, dz_z = max |dy| / |y| (+inf where y = 0 != dy), ymin = min |y|} (d null: ones; NaN wins)
constexpr int NSTAT = REFINE_NSTAT;
__global__ void __launch_bounds__(MAXT) column_stats_kernel(const double* __restrict__ Y, const double* __restrict__ DY,
                                                            const double* __restrict__ d, int M, int ldn,
                                                            double* __restrict__ out) {
    __shared__ double sh[NSTAT][MAXT];
    const int c = blockIdx.x;
    auto mx = [](double a, double b) { return (b > a || b != b) ? b : a; };
    auto mn = [](double a, double b) { return (b < a || b != b) ? b : a; };
    double v[NSTAT] = {0.0, 0.0, 0.0, 0.0, INFINITY};
    for (int i = threadIdx.x; i < M; i += MAXT) {
        const double yk = fabs(Y[(int64_t)i * ldn + c]), dyk = fabs(DY[(int64_t)i * ldn + c]), di = d ? d[i] : 1.0;
        v[0] = mx(v[0], yk);
        v[1] = mx(v[1], d ? yk * di : yk);
        v[2] = mx(v[2], d ? dyk * di : dyk);
        v[3] = mx(v[3], yk != 0.0 ? dyk / yk : dyk != 0.0 ? INFINITY : 0.0);
        v[4] = mn(v[4], yk);
    }
#pragma unroll
    for (int q = 0; q < NSTAT; ++q) sh[q][threadIdx.x] = v[q];
    __syncthreads();
    for (int w = MAXT / 2; w > 0; w >>= 1) {
        if (threadIdx.x < w) {
#pragma unroll
            for (int q = 0; q < NSTAT - 1; ++q) sh[q][threadIdx.x] = mx(sh[q][threadIdx.x], sh[q][threadIdx.x + w]);
            sh[4][threadIdx.x] = mn(sh[4][threadIdx.x], sh[4][threadIdx.x + w]);
        }
        __syncthreads();
    }
    if (threadIdx.x < NSTAT) out[(int64_t)c * NSTAT + threadIdx.x] = sh[threadIdx.x][0];
}

// refine_x's update of column c by how[c]: 1 y += dy; 2 (y, y_tail) += dy as LAPACK dla_wwaddw; 0 nothing
__global__ void update_x_kernel(double* __restrict__ Y, double* __restrict__ T, const double* __restrict__ DY,
                                const int* __restrict__ how, int M, int ldn) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (int64_t)M * ldn) return;
    const int h = how[e % ldn];
    if (h == 1) {
        Y[e] = __dadd_rn(Y[e], DY[e]);
    } else if (h == 2) {
        const double x = Y[e], w = DY[e];
        double s = __dadd_rn(x, w);
        s = __dsub_rn(__dadd_rn(s, s), s);
        double t = __dadd_rn(__dadd_rn(__dsub_rn(x, s), w), T[e]);
        const double xn = __dadd_rn(s, t);
        T[e] = __dadd_rn(__dsub_rn(s, xn), t);
        Y[e] = xn;
    }
}
}  // namespace

void refine_safe(int M, double* safe1, double* safe2, double* nzeps) {
    const double eps = std::ldexp(1.0, -53), safmin = std::ldexp(1.0, -1022);
    const double nz = (double)M + 1.0;
    *safe1 = nz * safmin;
    *safe2 = *safe1 / eps;
    *nzeps = nz * eps;
}
int launch_assemble(const AssembleArgs& a, bool extended, cudaStream_t s) {
    const dim3 grid((unsigned)a.M, (unsigned)((a.nrhs + 127) / 128));
    if (extended) assemble_x_kernel<<<grid, 128, 0, s>>>(a);
    else assemble_kernel<<<grid, 128, 0, s>>>(a);
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}
int launch_column_max(const double* ratio, int M, int ldn, int nrhs, double* berr, cudaStream_t s) {
    column_max_kernel<<<nrhs, MAXT, 0, s>>>(ratio, M, ldn, berr);
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}
int launch_column_stats(const double* Y, const double* DY, const double* d, int M, int ldn, int nrhs, double* out,
                        cudaStream_t s) {
    column_stats_kernel<<<nrhs, MAXT, 0, s>>>(Y, DY, d, M, ldn, out);
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}
static unsigned refine_blocks(int M, int ldn) { return (unsigned)(((size_t)M * ldn + 255) / 256); }
int launch_select_cols(const double* in, const int* active, int M, int ldn, double* out, cudaStream_t s) {
    select_cols_kernel<<<refine_blocks(M, ldn), 256, 0, s>>>(in, active, M, ldn, out);
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}
int launch_add_cols(double* X, const double* D, const int* active, int M, int ldn, cudaStream_t s) {
    add_cols_kernel<<<refine_blocks(M, ldn), 256, 0, s>>>(X, D, active, M, ldn);
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}
int launch_update_x(double* Y, double* T, const double* DY, const int* how, int M, int ldn, cudaStream_t s) {
    update_x_kernel<<<refine_blocks(M, ldn), 256, 0, s>>>(Y, T, DY, how, M, ldn);
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}

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

int launch_residual_x(ResidMode mode, const double* A, const Layout& L, const double* Xc, const double* Xct,
                      const double* Xr, const double* Xrt, int64_t ldx, int nrhs, double* Hi, double* Lo, int64_t ldo,
                      cudaStream_t s) {
    if (nrhs <= 0) return CFLX_OK;
    const int64_t lda = L.Nl;
    const int Ml = L.Ml, Nl = L.Nl, v = L.v;
    const ResidXArgs nn{Ml, nrhs, Nl, A, lda, Xc, Xct, ldx, Hi, Lo, ldo, v, L.Nt, MASK_NONE, L.Px, L.pi, L.Py, L.pj};
    const ResidXArgs tn{Nl, nrhs, Ml, A, lda, Xr, Xrt, ldx, Hi, Lo, ldo, v, L.Nt, MASK_NONE, L.Py, L.pj, L.Px, L.pi};
    if (mode == ResidMode::NN) return dispatch_x(nn, false, s);
    if (mode == ResidMode::TN) return dispatch_x(tn, true, s);
    ResidXArgs n2 = nn, t2 = tn;
    n2.mask = MASK_LOWER;
    t2.mask = MASK_STRICT_UPPER_T;
    t2.Hi = Hi + (int64_t)Ml * ldo;
    t2.Lo = Lo + (int64_t)Ml * ldo;
    CFLX_TRY(dispatch_x(n2, false, s));
    return dispatch_x(t2, true, s);
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

// ---------------------------------------------------------------- the refinement drivers
namespace {
// What both drivers share: the gather maps and the buffers for nrhs columns, X and B uploaded, and one residual pass.
struct RefinePass {
    RefineCache* rc;
    const RefineOp& op;
    int nrhs, ldn;
    bool nn, tn, layer0;
    size_t mat, chunk;
    AssembleArgs aa;
    std::vector<double> berr;

    RefinePass(RefineCache* rc_, const RefineOp& op_, int nrhs_) : rc(rc_), op(op_), nrhs(nrhs_), berr(nrhs_) {
        const Grid& G = op.grid;
        ldn = (int)round_up(nrhs, 8);
        nn = op.mode != ResidMode::TN;
        tn = op.mode != ResidMode::NN;
        layer0 = G.pk == 0;
        mat = (size_t)G.M * ldn;
        chunk = (size_t)((nn ? G.Ml : 0) + (tn ? G.Nl : 0)) * 2 * ldn;
    }

    // extended: the tail of X and its gathered copies, the per-column statistics and the update selector
    int setup(const double* B, int ldb, const double* X, int ldx, bool extended) {
        const Grid& G = op.grid;
        cflx_comm* c = G.comm;
        cudaStream_t s = c->stream;
        const int M = G.M, Ml = G.Ml, Nl = G.Nl;
        // local column (by_col) or row -> global row of X (clamped into X: masked entries never use the value)
        auto make_map = [&](DevBuf<int>* dst, int n, bool by_col) -> int {
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
        CFLX_TRY(grow_together({&rc->X, &rc->B, &rc->R, &rc->D, &rc->rhs, &rc->ratio, &rc->W}, mat));
        CFLX_TRY(rc->Xc.grow((size_t)Nl * ldn));
        CFLX_TRY(rc->Xr.grow((size_t)Ml * ldn));
        CFLX_TRY(rc->part.grow(chunk));
        if (c->world_size > 1) CFLX_TRY(rc->all.grow(chunk * c->world_size));
        CFLX_TRY(rc->berr.grow((size_t)ldn));
        CFLX_TRY(rc->active.grow((size_t)ldn));
        if (extended) {
            CFLX_TRY(rc->T.grow(mat));
            CFLX_TRY(rc->Xct.grow((size_t)Nl * ldn));
            CFLX_TRY(rc->Xrt.grow((size_t)Ml * ldn));
            CFLX_TRY(rc->stats.grow((size_t)ldn * NSTAT));
            CFLX_CUDA(cudaMemsetAsync(rc->T, 0, sizeof(double) * mat, s));
        }
        CFLX_CUDA(cudaMemsetAsync(rc->X, 0, sizeof(double) * mat, s));
        CFLX_CUDA(cudaMemsetAsync(rc->B, 0, sizeof(double) * mat, s));
        CFLX_CUDA(cudaMemcpy2DAsync(rc->X, ldn * sizeof(double), X, (size_t)ldx * sizeof(double), nrhs * sizeof(double), M,
                                    cudaMemcpyDefault, s));
        CFLX_CUDA(cudaMemcpy2DAsync(rc->B, ldn * sizeof(double), B, (size_t)ldb * sizeof(double), nrhs * sizeof(double), M,
                                    cudaMemcpyDefault, s));
        double safe1, safe2, nzeps;
        refine_safe(M, &safe1, &safe2, &nzeps);
        const double* all = c->world_size > 1 ? rc->all : rc->part;
        aa = AssembleArgs{all, (int64_t)chunk, Ml, Nl, ldn, nrhs, M, nn, tn, G.v, G.Px, G.Py, G.Pz, rc->B, rc->R,
                          rc->ratio, rc->W, safe1, safe2, nzeps};
        return CFLX_OK;
    }

    // the partials of op(A) (X + T) of every layer-0 rank on every rank (T: the tail, extended passes only)
    int partials(const double* X, const double* T) {
        const Grid& G = op.grid;
        cflx_comm* c = G.comm;
        cudaStream_t s = c->stream;
        if (layer0) {
            if (nn) CFLX_TRY(launch_gather_rows(X, ldn, rc->gl_cols, G.Nl, ldn, rc->Xc, s));
            if (tn) CFLX_TRY(launch_gather_rows(X, ldn, rc->gl_rows, G.Ml, ldn, rc->Xr, s));
            if (T) {
                if (nn) CFLX_TRY(launch_gather_rows(T, ldn, rc->gl_cols, G.Nl, ldn, rc->Xct, s));
                if (tn) CFLX_TRY(launch_gather_rows(T, ldn, rc->gl_rows, G.Ml, ldn, rc->Xrt, s));
                CFLX_TRY(launch_residual_x(op.mode, op.A, G, rc->Xc, rc->Xct, rc->Xr, rc->Xrt, ldn, nrhs, rc->part,
                                           rc->part + ldn, 2 * (int64_t)ldn, s));
            } else {
                CFLX_TRY(launch_residual(op.mode, op.A, G, rc->Xc, rc->Xr, ldn, nrhs, rc->part, rc->part + ldn,
                                         2 * (int64_t)ldn, s));
            }
        }
        if (c->world_size > 1) CFLX_NCCL(ncclAllGather(rc->part, rc->all, chunk, ncclDouble, c->world, s));
        return CFLX_OK;
    }

    // one working-precision pass over X (M x ldn): R = B - op(A) X, the ratios (and W, or Q when lin_berr), and the
    // per-column maximum ratio into berr on the host
    int run(const double* X, bool lin_berr = false, double* Q = nullptr) {
        cudaStream_t s = op.grid.comm->stream;
        CFLX_TRY(partials(X, nullptr));
        AssembleArgs a = aa;
        a.lin_berr = lin_berr;
        a.Q = Q;
        CFLX_TRY(launch_assemble(a, false, s));
        CFLX_TRY(launch_column_max(rc->ratio, op.grid.M, ldn, nrhs, rc->berr, s));
        CFLX_CUDA(cudaMemcpyAsync(berr.data(), rc->berr, sizeof(double) * nrhs, cudaMemcpyDeviceToHost, s));
        CFLX_CUDA(cudaStreamSynchronize(s));
        return CFLX_OK;
    }

    // R = B - op(A) (X + T) in double-double, rounded once
    int run_x() {
        cudaStream_t s = op.grid.comm->stream;
        CFLX_TRY(partials(rc->X, rc->T));
        return launch_assemble(aa, true, s);
    }

    // D = inv(op A) R on the columns where active (the others get 0)
    int correction(const std::vector<int>& active) {
        cudaStream_t s = op.grid.comm->stream;
        CFLX_CUDA(cudaMemcpyAsync(rc->active, active.data(), sizeof(int) * ldn, cudaMemcpyHostToDevice, s));
        CFLX_TRY(launch_select_cols(rc->R, rc->active, op.grid.M, ldn, rc->rhs, s));
        return op.solve(false, nrhs, rc->rhs, ldn, rc->D, ldn);  // synchronises: `active` may change after it
    }

    unsigned blocks() const { return (unsigned)((mat + 255) / 256); }
};

// dlacn2 on every column j with want[j], all in lockstep: a round issues one solve per kind over the columns that ask for
// it.  Column j estimates the 1-norm of diag(l_j) inv(op A)^T diag(r_j) (kase 1) / diag(r_j) inv(op A) diag(l_j) (kase
// 2): l and r are host M x ld arrays (r may be null: ones; where r_div[j], r_j is applied by division, as LAPACK's
// dla_gercond applies inv(C) with CMODE 1).  est[j] = the estimate (0 where not wanted).
int lacn2_columns(const RefineOp& op, int ncols, int ld, const std::vector<double>& l, const std::vector<double>* r,
                  const std::vector<char>* r_div, const std::vector<char>& want, std::vector<double>& est_out) {
    const int M = op.grid.M;
    std::vector<Lacn2> est(ncols);
    for (int j = 0; j < ncols; ++j)
        if (want[j]) est[j].start(M);
    auto R = [&](size_t o, double x) { return !r ? x : (*r_div)[o % ld] ? x / (*r)[o] : x * (*r)[o]; };
    std::vector<double> in((size_t)M * ld), out((size_t)M * ld);
    auto solve_round = [&](bool transposed, bool want1, bool want2) -> int {
        bool any = false;
        std::fill(in.begin(), in.end(), 0.0);
        for (int j = 0; j < ncols; ++j) {
            const int k = est[j].kase;
            if (!((k == 1 && want1) || (k == 2 && want2))) continue;
            any = true;
            for (int i = 0; i < M; ++i) {
                const size_t o = (size_t)i * ld + j;
                in[o] = k == 2 ? l[o] * est[j].x[i] : R(o, est[j].x[i]);
            }
        }
        if (!any) return CFLX_OK;
        CFLX_TRY(op.solve(transposed, ncols, in.data(), ld, out.data(), ld));
        for (int j = 0; j < ncols; ++j) {
            const int k = est[j].kase;
            if (!((k == 1 && want1) || (k == 2 && want2))) continue;
            for (int i = 0; i < M; ++i) {
                const size_t o = (size_t)i * ld + j;
                est[j].x[i] = k == 1 ? l[o] * out[o] : R(o, out[o]);
            }
            est[j].pending = true;
        }
        return CFLX_OK;
    };
    for (;;) {
        bool any = false;
        for (int j = 0; j < ncols; ++j) any |= est[j].kase != 0;
        if (!any) break;
        if (op.symmetric) {
            CFLX_TRY(solve_round(false, true, true));
        } else {
            CFLX_TRY(solve_round(true, true, false));
            CFLX_TRY(solve_round(false, false, true));
        }
        for (int j = 0; j < ncols; ++j)
            if (est[j].pending) {
                est[j].pending = false;
                est[j].step();
            }
    }
    est_out.assign(ncols, 0.0);
    for (int j = 0; j < ncols; ++j) est_out[j] = est[j].est;
    return CFLX_OK;
}
}  // namespace

int refine_run(RefineCache* rc, const RefineOp& op, int nrhs, const double* B, int ldb, double* X, int ldx, double* ferr,
               double* berr_out) {
    cudaStream_t s = op.grid.comm->stream;
    const int M = op.grid.M;
    RefinePass pass(rc, op, nrhs);
    CFLX_TRY(pass.setup(B, ldb, X, ldx, false));
    const int ldn = pass.ldn;
    const size_t mat = pass.mat;
    const std::vector<double>& berr = pass.berr;
    const double eps = std::ldexp(1.0, -53);

    // dgerfs, every column in lockstep: iterate while berr > eps, berr <= lstres / 2 and count <= ITMAX
    constexpr int ITMAX = 5;
    std::vector<int> count(nrhs, 1), active(ldn, 0);
    std::vector<double> lstres(nrhs, 3.0), col_berr(nrhs, 0.0);
    std::vector<char> refining(nrhs, 1);
    for (;;) {
        CFLX_TRY(pass.run(rc->X));
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
        CFLX_TRY(pass.correction(active));
        CFLX_TRY(launch_add_cols(rc->X, rc->D, rc->active, M, ldn, s));
    }
    std::vector<double> hX(mat);
    CFLX_CUDA(cudaMemcpyAsync(hX.data(), rc->X, sizeof(double) * mat, cudaMemcpyDeviceToHost, s));
    CFLX_CUDA(cudaStreamSynchronize(s));

    if (ferr) {
        // ||inv(op A)| w|_inf by dlacn2 on diag(w) inv(op A)^T (kase 1) and inv(op A) diag(w) (kase 2), one estimator per
        // column
        std::vector<double> w(mat), est;
        CFLX_CUDA(cudaMemcpyAsync(w.data(), rc->W, sizeof(double) * mat, cudaMemcpyDeviceToHost, s));
        CFLX_CUDA(cudaStreamSynchronize(s));
        CFLX_TRY(lacn2_columns(op, nrhs, ldn, w, nullptr, nullptr, std::vector<char>(nrhs, 1), est));
        for (int j = 0; j < nrhs; ++j) {
            double xmax = 0.0;
            for (int i = 0; i < M; ++i) xmax = std::max(xmax, std::fabs(hX[(size_t)i * ldn + j]));
            ferr[j] = xmax != 0.0 ? est[j] / xmax : est[j];
        }
    }
    CFLX_CUDA(cudaMemcpy2DAsync(X, (size_t)ldx * sizeof(double), rc->X, ldn * sizeof(double), nrhs * sizeof(double), M,
                                cudaMemcpyDefault, s));
    CFLX_CUDA(cudaStreamSynchronize(s));
    if (berr_out) std::copy(col_berr.begin(), col_berr.end(), berr_out);
    return CFLX_OK;
}

// ---------------------------------------------------------------- extra-precise refinement (dgerfsx / dporfsx)
int RefineXColumn::round(const double st[5], double rcond, bool ignore_cwise, int cnt, int M) {
    const double eps = std::ldexp(1.0, -53), incr_thresh = (double)M * eps;
    constexpr double RTHRESH = 0.5, DZ_UB = 0.25;
    const double normy = st[0], normx = st[1], normdx = st[2], ymin = st[4];
    dz_z = st[3];
    dx_x = normx != 0.0 ? normdx / normx : normdx == 0.0 ? 0.0 : INFINITY;
    const double dxrat = normdx / prev_normdx, dzrat = dz_z / prev_dz_z;
    bool incr_prec = !ignore_cwise && ymin * rcond < incr_thresh * normy && y_prec < EXTRA_Y;

    if (x_state == NOPROG && dxrat <= RTHRESH) x_state = WORKING;
    if (x_state == WORKING) {
        if (dx_x <= eps) {
            x_state = CONV;
        } else if (dxrat > RTHRESH) {
            if (y_prec != EXTRA_Y) incr_prec = true;
            else x_state = NOPROG;
        } else if (dxrat > dxratmax) {
            dxratmax = dxrat;
        }
        if (x_state > WORKING) final_dx_x = dx_x;
    }
    if (z_state == UNSTABLE && dz_z <= DZ_UB) z_state = WORKING;
    if (z_state == NOPROG && dzrat <= RTHRESH) z_state = WORKING;
    if (z_state == WORKING) {
        if (dz_z <= eps) {
            z_state = CONV;
        } else if (dz_z > DZ_UB) {
            z_state = UNSTABLE;
            dzratmax = 0.0;
            final_dz_z = INFINITY;
        } else if (dzrat > RTHRESH) {
            if (y_prec != EXTRA_Y) incr_prec = true;
            else z_state = NOPROG;
        } else if (dzrat > dzratmax) {
            dzratmax = dzrat;
        }
        if (z_state > WORKING) final_dz_z = dz_z;
    }
    if (x_state != WORKING &&
        (ignore_cwise || z_state == NOPROG || z_state == CONV || (z_state == UNSTABLE && cnt > 1))) {
        done = true;
        return 0;
    }
    if (incr_prec) y_prec = EXTRA_Y;  // the tail is zero until the first double-double update
    prev_normdx = normdx;
    prev_dz_z = dz_z;
    return y_prec == EXTRA_Y ? 2 : 1;
}

void RefineXColumn::finish() {
    if (x_state == WORKING) final_dx_x = dx_x;
    if (z_state == WORKING) final_dz_z = dz_z;
    err_norm = final_dx_x / (1.0 - dxratmax);
    err_comp = final_dz_z / (1.0 - dzratmax);
}

int refine_x_run(RefineCache* rc, const RefineOp& op, int nrhs, const double* B, int ldb, double* X, int ldx,
                 const double* d, double rcond, bool cwise, double* berr_out, double* err_norm, double* err_comp,
                 int* info) {
    cudaStream_t s = op.grid.comm->stream;
    const int M = op.grid.M;
    RefinePass pass(rc, op, nrhs);
    CFLX_TRY(pass.setup(B, ldb, X, ldx, true));
    const int ldn = pass.ldn;
    const size_t mat = pass.mat;
    constexpr int ITHRESH = 10;

    // dla_gerfsx_extended / dla_porfsx_extended, every column in lockstep from the extra-residual state
    std::vector<RefineXColumn> col(nrhs);
    std::vector<int> active(ldn, 0), how(ldn, 0);
    std::vector<double> st((size_t)ldn * NSTAT);
    for (int cnt = 1; cnt <= ITHRESH; ++cnt) {
        bool any = false;
        for (int j = 0; j < nrhs; ++j) any |= (active[j] = !col[j].done) != 0;
        if (!any) break;
        CFLX_TRY(pass.run_x());
        CFLX_TRY(pass.correction(active));
        CFLX_TRY(launch_column_stats(rc->X, rc->D, d, M, ldn, nrhs, rc->stats, s));
        CFLX_CUDA(cudaMemcpyAsync(st.data(), rc->stats, sizeof(double) * nrhs * NSTAT, cudaMemcpyDeviceToHost, s));
        CFLX_CUDA(cudaStreamSynchronize(s));
        for (int j = 0; j < nrhs; ++j) how[j] = active[j] ? col[j].round(&st[(size_t)j * NSTAT], rcond, !cwise, cnt, M) : 0;
        CFLX_CUDA(cudaMemcpyAsync(rc->active, how.data(), sizeof(int) * ldn, cudaMemcpyHostToDevice, s));
        CFLX_TRY(launch_update_x(rc->X, rc->T, rc->D, rc->active, M, ldn, s));
    }
    for (RefineXColumn& c : col) c.finish();

    // berr (dla_lin_berr) from one working-precision pass, which also gives |op(A)| |y| for the componentwise condition
    CFLX_TRY(pass.run(rc->X, true, rc->W));
    std::vector<double> hY(mat), ayq;
    CFLX_CUDA(cudaMemcpyAsync(hY.data(), rc->X, sizeof(double) * mat, cudaMemcpyDeviceToHost, s));
    if (cwise) {
        ayq.resize(mat);
        CFLX_CUDA(cudaMemcpyAsync(ayq.data(), rc->W, sizeof(double) * mat, cudaMemcpyDeviceToHost, s));
    }
    CFLX_CUDA(cudaStreamSynchronize(s));
    if (berr_out) std::copy(pass.berr.begin(), pass.berr.end(), berr_out);

    // The condition estimates, all in lockstep: column j < nrhs the componentwise one of y_j (dla_gercond CMODE 1:
    // l = |op(A)| |y_j|, applied with inv(diag(y_j))), where its bound is below sqrt(eps); column nrhs the normwise one
    // of op(A) inv(diag(d)) (CMODE -1: l = |op(A)| |1 / d|, applied with diag(d); CMODE 0 without d: l = |op(A)| 1).
    const int ncols = nrhs + 1, ld = (int)round_up(ncols, 8);
    std::vector<double> l((size_t)M * ld, 0.0), r((size_t)M * ld, 1.0);
    std::vector<char> want(ncols, 0), r_div(ld, 1);
    const double eps = std::ldexp(1.0, -53), cwise_wrong = std::sqrt(eps);
    {
        // |op(A)| |1 / d| by one more working-precision pass with 1 / d (or ones) in column 0
        std::vector<double> hd(M, 1.0), one(mat, 0.0);
        if (d) {
            CFLX_CUDA(cudaMemcpyAsync(hd.data(), d, sizeof(double) * M, cudaMemcpyDeviceToHost, s));
            CFLX_CUDA(cudaStreamSynchronize(s));
        }
        for (int i = 0; i < M; ++i) one[(size_t)i * ldn] = d ? 1.0 / hd[i] : 1.0;
        CFLX_CUDA(cudaMemcpyAsync(rc->rhs, one.data(), sizeof(double) * mat, cudaMemcpyHostToDevice, s));
        CFLX_TRY(pass.run(rc->rhs, true, rc->W));
        std::vector<double> g(mat);
        CFLX_CUDA(cudaMemcpyAsync(g.data(), rc->W, sizeof(double) * mat, cudaMemcpyDeviceToHost, s));
        CFLX_CUDA(cudaStreamSynchronize(s));
        for (int i = 0; i < M; ++i) {
            l[(size_t)i * ld + nrhs] = g[(size_t)i * ldn];
            r[(size_t)i * ld + nrhs] = hd[i];
        }
        want[nrhs] = 1;
        r_div[nrhs] = 0;
    }
    if (cwise)
        for (int j = 0; j < nrhs; ++j) {
            want[j] = col[j].err_comp < cwise_wrong;
            for (int i = 0; i < M; ++i) {
                l[(size_t)i * ld + j] = ayq[(size_t)i * ldn + j];
                r[(size_t)i * ld + j] = hY[(size_t)i * ldn + j];
            }
        }
    std::vector<double> est;
    CFLX_TRY(lacn2_columns(op, ncols, ld, l, &r, &r_div, want, est));
    auto cond = [&](int j) { return est[j] != 0.0 ? 1.0 / est[j] : 0.0; };

    const double illrcond_thresh = (double)M * eps, err_lbnd = std::max(10.0, std::sqrt((double)M)) * eps;
    int first_ill = 0;
    auto bound = [&](double err, double rc_, int j, double* out) {
        double trust = 1.0;
        err = std::min(err, 1.0);
        if (rc_ < illrcond_thresh) {
            err = 1.0;
            trust = 0.0;
            if (!first_ill) first_ill = j + 1;
        } else if (err < err_lbnd) {
            err = err_lbnd;
        }
        out[3 * j] = trust;
        out[3 * j + 1] = err;
        out[3 * j + 2] = rc_;
    };
    const double rcond_norm = cond(nrhs);
    for (int j = 0; j < nrhs; ++j) {
        bound(col[j].err_norm, rcond_norm, j, err_norm);
        if (cwise) bound(col[j].err_comp, want[j] ? cond(j) : 0.0, j, err_comp);
    }
    *info = first_ill ? M + first_ill : 0;
    CFLX_CUDA(cudaMemcpy2DAsync(X, (size_t)ldx * sizeof(double), rc->X, ldn * sizeof(double), nrhs * sizeof(double), M,
                                cudaMemcpyDefault, s));
    CFLX_CUDA(cudaStreamSynchronize(s));
    return CFLX_OK;
}

}  // namespace cflx
