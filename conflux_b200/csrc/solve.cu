// conflux_b200/csrc/solve.cu -- the triangular-solve engine of cflx_lu_solve (lu.cu) and cflx_chol_solve (chol.cu).
//
// A factor in the conflux block-cyclic layout (SolveFactor: tile (I, J) on rank (I % Px, J % Py, 0)) is solved against
// a few right-hand sides by sweeps over the tile diagonal.  In the row-partial sweep every rank keeps a partial
// right-hand side W (Ml x ldn, by local tile row); its sum over a grid row is the current right-hand side of those tile
// rows.  Step t:
//   ncclReduce of tile t's rows of W over the grid row onto the diagonal owner (t % Px, t % Py, 0);
//   the owner solves with the diagonal tile by an nb-block sweep with the inverses of its nb x nb diagonal blocks, and
//   keeps the solved tile where its caller asks;
//   ncclBroadcast of the solved tile over the grid column;
//   every layer-0 rank of that grid column updates its rows of the tiles past t.
// The column-partial sweep (L^T X = Y with only L stored) is the transpose: partials Z by local tile column, the reduce
// over the grid column, the broadcast over the grid row, and the update read transposed in place.  The owners write
// X_t into a zeroed M x ldn buffer, and one all-reduce makes X identical on every rank.  All arithmetic is the narrow
// GEMM below: a factor block (row-major, read in place) times a few right-hand sides.
#include <cmath>
#include <cstring>

#include "lu_state.h"
#include "narrow.cuh"

namespace cflx {
namespace {

// ---------------------------------------------------------------- the narrow GEMM
// D = beta * C + alpha * A * B, A [M x K] row-major (lda), B [K x N], C / D [M x N].  The workload is memory-bound on A
// (K = v or nb, N = a few right-hand sides), so every element of A is loaded exactly once per slab of BN columns, with
// 16-byte loads straight into the MMA fragments:
//   * a warp owns 16 rows x BN columns; lane (g = lane >> 2, t = lane & 3) loads A[g][k0 + 4t .. 4t+3] and
//     A[g+8][k0 + 4t .. 4t+3] of every 16-wide k step as two double2 each (a quad reads one 128-byte row segment);
//   * the k step is two mma.sync.m16n8k8.f64 whose k slots are permuted: in MMA h, slot t is k = 4t + 2h and slot t + 4 is
//     k = 4t + 2h + 1, so the two halves of one double2 feed the two k slots of one lane.  B is staged in shared memory
//     as k pairs, sB[k / 2][n] = {B[k][n], B[k + 1][n]}, so each B fragment is one 16-byte load;
//   * A is loaded one chunk at a time into registers (64 of them).  Loading it one chunk ahead needs KC = 32 to fit the
//     registers at BN = 64, and measured slower in the solve (4.8 against 4.1 ms at C2, one right-hand side): the
//     diagonal sweeps' 128-row GEMMs then run twice as many latency-bound chunks;
//   * B goes through shared memory in chunks of KC k rows, double-buffered: the 8-byte asynchronous copies (cp.async,
//     zero-filled beyond K and N) of chunk c + 1 are issued before chunk c is computed, so staging B costs no register
//     and no round trip on the critical path.  Staging B with plain loads and stores was 5x slower at BN = 64: a thread's
//     16 dependent L2 round trips per chunk were the whole kernel time.
// K % 4 == 0 is the only shape condition: a lane's four k indices are either all in range or all out of it, and both A
// (masked loads) and B (zero-filled staging) are zero beyond K, so nothing stale or NaN reaches the MMA.
// epilogue of one m16n8 tile row pair: acc[j][0..1] = D[row_a][n0 + 8j + 2t + {0,1}], acc[j][2..3] the same of row_b.  C
// may alias D: each element is read and then written by the same thread, so plain (coherent) accesses suffice.
template <int NT>
__device__ __forceinline__ void store_d(const NarrowArgs& g, const double (&acc)[NT][4], int64_t row_a, int64_t row_b,
                                        int n0, int t4) {
    const bool use_c = g.beta != 0.0;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int64_t row = r ? row_b : row_a;
        if (row >= g.M) continue;
#pragma unroll
        for (int j = 0; j < NT; ++j) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int col = n0 + 8 * j + 2 * t4 + e;
                if (col < g.N) {
                    const double c = use_c ? g.C[row * g.ldc + col] : 0.0;
                    g.D[row * g.ldd + col] = fma(g.alpha, acc[j][2 * r + e], g.beta * c);
                }
            }
        }
    }
}

template <int NT>
__global__ void __launch_bounds__(NW * 32, 1) gemm_narrow_kernel(NarrowArgs g) {
    constexpr int BN = NarrowCfg<NT>::BN, LDP = NarrowCfg<NT>::LDP, STEPS = KC / 16;
    extern __shared__ double2 sB[];  // [2][KC / 2][LDP]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g4 = lane >> 2, t4 = lane & 3;
    const int64_t row0 = (int64_t)blockIdx.x * BM + warp * 16 + g4;
    const int n0 = blockIdx.y * BN;
    const bool ok0 = row0 < g.M, ok1 = row0 + 8 < g.M;
    const double* a0p = g.A + (ok0 ? row0 * g.lda : 0);
    const double* a1p = g.A + (ok1 ? (row0 + 8) * g.lda : 0);
    double acc[NT][4];
#pragma unroll
    for (int j = 0; j < NT; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.0;

    // a[s][0..1] = row g, k 4t..4t+1 / 4t+2..4t+3 of step s of a chunk;  a[s][2..3] = the same of row g + 8
    auto load_a = [&](double2 (&a)[STEPS][4], int kc) {
#pragma unroll
        for (int s = 0; s < STEPS; ++s) {
            const int k = kc + 16 * s + 4 * t4;
            const bool kin = k < g.K;
            const double2 z = make_double2(0.0, 0.0);
            a[s][0] = (ok0 && kin) ? __ldg(reinterpret_cast<const double2*>(a0p + k)) : z;
            a[s][1] = (ok0 && kin) ? __ldg(reinterpret_cast<const double2*>(a0p + k + 2)) : z;
            a[s][2] = (ok1 && kin) ? __ldg(reinterpret_cast<const double2*>(a1p + k)) : z;
            a[s][3] = (ok1 && kin) ? __ldg(reinterpret_cast<const double2*>(a1p + k + 2)) : z;
        }
    };
    if (g.K > 0) stage_b<NT>(g, 0, n0, sB);
    for (int kc = 0, c = 0; kc < g.K; kc += KC, ++c) {
        double2 a[STEPS][4];
        load_a(a, kc);  // in flight while the chunk's B lands
        cp_async_wait_all();  // chunk c has landed (this thread's copies) ...
        __syncthreads();      // ... for every thread, and every warp is done with chunk c - 1's buffer
        if (kc + KC < g.K) stage_b<NT>(g, kc + KC, n0, sB + ((c + 1) & 1) * NarrowCfg<NT>::STAGE);
        const double2* sb = sB + (c & 1) * NarrowCfg<NT>::STAGE;
#pragma unroll
        for (int s = 0; s < STEPS; ++s) {
            if (kc + 16 * s < g.K) {  // uniform over the CTA
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const double af[4] = {a[s][h].x, a[s][2 + h].x, a[s][h].y, a[s][2 + h].y};
                    const double2* b_k = sb + (8 * s + 2 * t4 + h) * LDP + g4;
#pragma unroll
                    for (int j = 0; j < NT; ++j) {
                        const double2 bb = b_k[8 * j];
                        const double bf[2] = {bb.x, bb.y};
                        dmma16x8x8(acc[j], af, bf);
                    }
                }
            }
        }
    }

    // epilogue: c0/c1 = D[g][2t + {0,1}], c2/c3 = D[g + 8][2t + {0,1}] of every 8-column tile
    store_d<NT>(g, acc, row0, row0 + 8, n0, t4);
}

template <int NT>
int launch_narrow_nt(const NarrowArgs& g, cudaStream_t s) {
    using C = NarrowCfg<NT>;
    static PerDeviceMax cfg;
    CFLX_CUDA(cfg.raise(C::SMEM, [&] {
        return cudaFuncSetAttribute(gemm_narrow_kernel<NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM);
    }));
    dim3 grid((unsigned)((g.M + BM - 1) / BM), (unsigned)((g.N + C::BN - 1) / C::BN));
    gemm_narrow_kernel<NT><<<grid, NW * 32, C::SMEM, s>>>(g);
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}

// ---------------------------------------------------------------- the transposed narrow GEMM
// D = beta * C + alpha * AT^T * B, AT [K x M] row-major (NarrowArgs::A / lda), read in place: the backward sweep of the
// Cholesky solve applies L^T with only L stored.  Bound by reading AT like the kernel above, so every element of AT is
// loaded once per slab of BN columns, with 16-byte loads straight into the MMA fragments.  AT is contiguous in m, so one
// double2 holds two output rows of one k:
//   * a warp owns 32 rows m0 .. m0 + 31; lane (g, t) loads AT[k][m0 + 2g .. 2g+1] and AT[k][m0 + 16 + 2g .. 2g+1] for
//     the four k = 4t .. 4t+3 of every 16-wide k step (the eight lanes of one t read one 128-byte segment of a k row);
//   * MMA p in {0, 1} takes component p of every double2: row slot g is m0 + 2g + p and row slot g + 8 is
//     m0 + 16 + 2g + p.  The epilogue un-permutes by storing the two MMAs' tiles at those rows (store_d);
//   * the k slots are permuted as in the NN kernel (in MMA half h, slot t is k = 4t + 2h and slot t + 4 is k = 4t + 2h + 1),
//     so B is staged by the same stage_b and each B fragment is one conflict-free 16-byte shared-memory load;
//   * a 16-wide k step is 16 doubles of AT per lane against 8 * NT accumulators, so AT goes into registers KA k rows at a
//     time within each 64-row chunk of B (TnCfg: fewer rows as the accumulators grow, to stay clear of spills).
// No K condition: every k row is masked on its own and B is zero-filled beyond K and N.  With an odd M the last pair's
// second row is beyond M, and that pair is loaded as one double, so nothing beyond M, K or N is read.
constexpr int BM_TN = 32 * NW;  // rows per CTA

template <int NT>
struct TnCfg {
    static constexpr int KA = NT >= 8 ? 16 : (NT >= 4 ? 32 : 64);  // k rows of AT per register load
};

template <int NT>
__global__ void __launch_bounds__(NW * 32, 1) gemm_narrow_tn_kernel(NarrowArgs g) {
    constexpr int LDP = NarrowCfg<NT>::LDP, KA = TnCfg<NT>::KA, SUB = KA / 16;
    extern __shared__ double2 sB[];  // [2][KC / 2][LDP]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g4 = lane >> 2, t4 = lane & 3;
    const int64_t ma = (int64_t)blockIdx.x * BM_TN + warp * 32 + 2 * g4, mb = ma + 16;
    const int n0 = blockIdx.y * NarrowCfg<NT>::BN;
    double acc[2][NT][4];
#pragma unroll
    for (int p = 0; p < 2; ++p)
#pragma unroll
        for (int j = 0; j < NT; ++j) acc[p][j][0] = acc[p][j][1] = acc[p][j][2] = acc[p][j][3] = 0.0;

    auto load_pair = [&](const double* row, int64_t m) -> double2 {  // AT[k][m .. m+1], zero beyond M
        if (m + 1 < g.M) return __ldg(reinterpret_cast<const double2*>(row + m));
        return make_double2(m < g.M ? __ldg(row + m) : 0.0, 0.0);
    };
    // a[s][2i + r] = AT[k][m_r .. m_r + 1] with k = kk + 16s + 4t + i, m_0 = m0 + 2g, m_1 = m0 + 16 + 2g
    auto load_a = [&](double2 (&a)[SUB][8], int kk) {
#pragma unroll
        for (int s = 0; s < SUB; ++s) {
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int k = kk + 16 * s + 4 * t4 + i;
                const double2 z = make_double2(0.0, 0.0);
                a[s][2 * i] = k < g.K ? load_pair(g.A + (int64_t)k * g.lda, ma) : z;
                a[s][2 * i + 1] = k < g.K ? load_pair(g.A + (int64_t)k * g.lda, mb) : z;
            }
        }
    };
    if (g.K > 0) stage_b<NT>(g, 0, n0, sB);
    for (int kc = 0, c = 0; kc < g.K; kc += KC, ++c) {
        const double2* sb = sB + (c & 1) * NarrowCfg<NT>::STAGE;
#pragma unroll 1
        for (int ks = 0; ks < KC && kc + ks < g.K; ks += KA) {  // uniform over the CTA
            double2 a[SUB][8];
            load_a(a, kc + ks);  // the first load of a chunk is in flight while the chunk's B lands
            if (ks == 0) {
                cp_async_wait_all();  // chunk c has landed (this thread's copies) ...
                __syncthreads();      // ... for every thread, and every warp is done with chunk c - 1's buffer
                if (kc + KC < g.K) stage_b<NT>(g, kc + KC, n0, sB + ((c + 1) & 1) * NarrowCfg<NT>::STAGE);
            }
#pragma unroll
            for (int s = 0; s < SUB; ++s) {
                if (kc + ks + 16 * s < g.K) {  // uniform over the CTA
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const double2 *k0 = a[s] + 4 * h, *k1 = a[s] + 4 * h + 2;  // k = 4t + 2h and 4t + 2h + 1
                        const double af0[4] = {k0[0].x, k0[1].x, k1[0].x, k1[1].x};
                        const double af1[4] = {k0[0].y, k0[1].y, k1[0].y, k1[1].y};
                        const double2* b_k = sb + ((ks >> 1) + 8 * s + 2 * t4 + h) * LDP + g4;
#pragma unroll
                        for (int j = 0; j < NT; ++j) {
                            const double2 bb = b_k[8 * j];
                            const double bf[2] = {bb.x, bb.y};
                            dmma16x8x8(acc[0][j], af0, bf);
                            dmma16x8x8(acc[1][j], af1, bf);
                        }
                    }
                }
            }
        }
    }
#pragma unroll
    for (int p = 0; p < 2; ++p) store_d<NT>(g, acc[p], ma + p, mb + p, n0, t4);
}

template <int NT>
int launch_narrow_tn(const NarrowArgs& g, cudaStream_t s) {
    using C = NarrowCfg<NT>;
    static PerDeviceMax cfg;
    CFLX_CUDA(cfg.raise(C::SMEM, [&] {
        return cudaFuncSetAttribute(gemm_narrow_tn_kernel<NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM);
    }));
    dim3 grid((unsigned)((g.M + BM_TN - 1) / BM_TN), (unsigned)((g.N + C::BN - 1) / C::BN));
    gemm_narrow_tn_kernel<NT><<<grid, NW * 32, C::SMEM, s>>>(g);
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}

// Linv[j][r][c] = LinvT[j][c][r] for the v / nb blocks of one diagonal tile
__global__ void transpose_blocks_kernel(const double* __restrict__ in, int nb, int64_t total, double* __restrict__ out) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= total) return;
    const int64_t blk = e / ((int64_t)nb * nb);
    const int r = (int)(e / nb % nb), c = (int)(e % nb);
    out[e] = in[blk * nb * nb + (int64_t)c * nb + r];
}
}  // namespace

int launch_gemm_narrow(int M, int N, int K, const double* A, int64_t lda, const double* B, int64_t ldb, const double* C,
                       int64_t ldc, double* D, int64_t ldd, double alpha, double beta, cudaStream_t stream) {
    if (M <= 0 || N <= 0) return CFLX_OK;
    if (K < 0 || (K & 3) || (lda & 1) || (reinterpret_cast<uintptr_t>(A) & 15)) {
        set_last_error("gemm_narrow: unsupported shape M=%d N=%d K=%d lda=%lld (need K %% 4 == 0, even lda, 16-byte aligned A)",
                       M, N, K, (long long)lda);
        return CFLX_ERR_UNSUPPORTED;
    }
    const NarrowArgs g{M, N, K, A, lda, B, ldb, C, ldc, D, ldd, alpha, beta};
    if (N <= 8) return launch_narrow_nt<1>(g, stream);
    if (N <= 16) return launch_narrow_nt<2>(g, stream);
    if (N <= 32) return launch_narrow_nt<4>(g, stream);
    return launch_narrow_nt<8>(g, stream);  // wider B: slabs of 64 columns, one per blockIdx.y
}

int launch_gemm_narrow_tn(int M, int N, int K, const double* AT, int64_t ldat, const double* B, int64_t ldb, const double* C,
                          int64_t ldc, double* D, int64_t ldd, double alpha, double beta, cudaStream_t stream) {
    if (M <= 0 || N <= 0) return CFLX_OK;
    if (K < 0 || (ldat & 1) || ldat < M || (reinterpret_cast<uintptr_t>(AT) & 15)) {
        set_last_error("gemm_narrow_tn: unsupported shape M=%d N=%d K=%d ldat=%lld (need K >= 0, even ldat >= M, 16-byte aligned AT)",
                       M, N, K, (long long)ldat);
        return CFLX_ERR_UNSUPPORTED;
    }
    const NarrowArgs g{M, N, K, AT, ldat, B, ldb, C, ldc, D, ldd, alpha, beta};
    if (N <= 8) return launch_narrow_tn<1>(g, stream);
    if (N <= 16) return launch_narrow_tn<2>(g, stream);
    if (N <= 32) return launch_narrow_tn<4>(g, stream);
    return launch_narrow_tn<8>(g, stream);
}

// ---------------------------------------------------------------- the solve engine
namespace {
int launch_transpose_blocks(const double* in, int nb, int64_t total, double* out, cudaStream_t stream) {
    transpose_blocks_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(in, nb, total, out);
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}

// slot of diagonal tile t in SolveCache::inv on this rank (-1: not owned)
int diag_slot(const SolveFactor& f, int t) {
    if (f.g.pk != 0 || t % f.g.Px != f.g.pi || t % f.g.Py != f.g.pj) return -1;
    int n = 0;
    for (int u = 0; u < t; ++u) n += (u % f.g.Px == f.g.pi && u % f.g.Py == f.g.pj);
    return n;
}

const double* diag_tile(const SolveFactor& f, int t) {
    return f.F + (int64_t)f.g.diag_row(t) * f.g.Nl + f.g.diag_col(t);
}

// diag_solve on the owner of diagonal tile t, with its cached inverses, into sc.Y
int diag_solve_tile(const SolveCache& sc, const SolveFactor& f, int t, Tri tri, double* R, int ldn, cudaStream_t s) {
    const double* inv = sc.inv + diag_slot(f, t) * 2 * (size_t)f.g.v * f.g.nb;
    return diag_solve(inv, diag_tile(f, t), f.g.Nl, f.g.v, f.g.nb, tri, R, sc.Y, ldn, s);
}
}  // namespace

int solve_tile_inverses(const double* T, int64_t ld, int v, int nb, bool lower, double* inv, double* tile, double* linvT,
                        cudaStream_t s) {
    // launch_diag_inverses takes an A00 = L\U.  A lower L goes in as L_tt^T, as the Cholesky panel step runs it:
    // Uinv_j = inv(L_jj)^T is then the backward half, its block transpose inv(L_jj) the forward half, and the
    // unit-lower part is the identity.  For L\U, the forward half is the block transpose of LinvT.
    if (lower) {
        CFLX_TRY(launch_extract_panel_T(T, ld, 0, 0, v, v, tile, v, s));
    } else if (cudaMemcpy2DAsync(tile, v * sizeof(double), T, ld * sizeof(double), v * sizeof(double), v,
                                 cudaMemcpyDeviceToDevice, s) != cudaSuccess) {
        set_last_error("solve: diagonal tile copy failed");
        return CFLX_ERR_CUDA;
    }
    CFLX_TRY(launch_diag_inverses(tile, v, nb, inv + (size_t)v * nb, linvT, s));
    return launch_transpose_blocks(lower ? inv + (size_t)v * nb : linvT, nb, (int64_t)v * nb, inv, s);
}

// Y = T^-1 R by an nb-block sweep with the cached inverses; R (v x ldn) is overwritten.
//   Lower:      T = L_tt:    Y_j = inv(L_jj) R_j, then R_i -= L_ij Y_j for i > j (the forward inverses)
//   Upper:      T = U_tt:    Y_j = inv(U_jj) R_j, then R_i -= U_ij Y_j for i < j (the backward inverses)
//   LowerT:     T = L_tt^T:  Y_j = inv(L_jj)^T R_j, then R_i -= L_ji^T Y_j for i < j (the backward inverses; L_tt read
//               transposed in place)
//   UnitLowerT: as LowerT, but inv(L_jj)^T is the forward inverse block read transposed (the LU's unit L)
//   UpperT:     T = U_tt^T:  Y_j = inv(U_jj)^T R_j (the backward inverse block read transposed), then R_i -= U_ji^T Y_j
//               for i > j: one TN launch on block row j of U_tt right of its diagonal block
int diag_solve(const double* tile_inv, const double* ftt, int64_t Nl, int v, int nb, Tri tri, double* R, double* Y,
               int ldn, cudaStream_t s) {
    const int nblk = v / nb;
    const bool fwd = tri == Tri::Lower, ascending = fwd || tri == Tri::UpperT;
    const bool fwd_half = fwd || tri == Tri::UnitLowerT, inv_tn = tri == Tri::UnitLowerT || tri == Tri::UpperT;
    const double* inv = tile_inv + (fwd_half ? 0 : (size_t)v * nb);
    for (int i = 0; i < nblk; ++i) {
        const int j = ascending ? i : nblk - 1 - i;
        const int64_t o = (int64_t)j * nb * ldn;
        if (inv_tn)
            CFLX_TRY(launch_gemm_narrow_tn(nb, ldn, nb, inv + (size_t)j * nb * nb, nb, R + o, ldn, nullptr, ldn, Y + o, ldn,
                                           1.0, 0.0, s));
        else
            CFLX_TRY(launch_gemm_narrow(nb, ldn, nb, inv + (size_t)j * nb * nb, nb, R + o, ldn, nullptr, ldn, Y + o, ldn,
                                        1.0, 0.0, s));
        if (fwd && j + 1 < nblk) {
            const int64_t o1 = (int64_t)(j + 1) * nb;
            CFLX_TRY(launch_gemm_narrow(v - (j + 1) * nb, ldn, nb, ftt + o1 * Nl + (int64_t)j * nb, Nl, Y + o, ldn,
                                        R + o1 * ldn, ldn, R + o1 * ldn, ldn, -1.0, 1.0, s));
        }
        if (tri == Tri::Upper && j > 0)
            CFLX_TRY(launch_gemm_narrow(j * nb, ldn, nb, ftt + (int64_t)j * nb, Nl, Y + o, ldn, R, ldn, R, ldn, -1.0, 1.0, s));
        if ((tri == Tri::LowerT || tri == Tri::UnitLowerT) && j > 0)  // block row j of L_tt left of its diagonal block, as AT
            CFLX_TRY(launch_gemm_narrow_tn(j * nb, ldn, nb, ftt + (int64_t)j * nb * Nl, Nl, Y + o, ldn, R, ldn, R, ldn,
                                           -1.0, 1.0, s));
        if (tri == Tri::UpperT && j + 1 < nblk) {  // block row j of U_tt right of its diagonal block, as AT
            const int64_t o1 = (int64_t)(j + 1) * nb;
            CFLX_TRY(launch_gemm_narrow_tn(v - (j + 1) * nb, ldn, nb, ftt + (int64_t)j * nb * Nl + o1, Nl, Y + o, ldn,
                                           R + o1 * ldn, ldn, R + o1 * ldn, ldn, -1.0, 1.0, s));
        }
    }
    return CFLX_OK;
}

int solve_cache_grow(SolveCache* sc, const SolveFactor& f, int ldn, bool work, bool col_partials, bool col_seed) {
    if (ldn <= sc->ldn && (sc->col_partials || !col_partials) && (sc->col_seed || !col_seed)) return CFLX_OK;
    ldn = std::max(ldn, sc->ldn);
    sc->col_partials |= col_partials;
    sc->col_seed |= col_seed;
    for (DevBuf<double>* p : {&sc->B, &sc->W, &sc->Z, &sc->R, &sc->Y, &sc->X, &sc->Xg}) p->reset();
    sc->ldn = 0;
    const size_t M = f.g.M, v = f.g.v;
    if (f.g.pk == 0 && (f.g.pj == 0 || (sc->col_seed && f.g.pi == 0))) CFLX_TRY(sc->B.alloc(M * ldn));
    if (work) {
        CFLX_TRY(sc->W.alloc((size_t)f.g.Ml * ldn));
        if (sc->col_partials) CFLX_TRY(sc->Z.alloc((size_t)f.g.Nl * ldn));
        CFLX_TRY(sc->R.alloc(v * ldn));
        CFLX_TRY(sc->Y.alloc(v * ldn));
    }
    CFLX_TRY(sc->X.alloc(M * ldn));
    if (sc->col_seed) CFLX_TRY(sc->Xg.alloc(M * ldn));
    sc->ldn = ldn;
    return CFLX_OK;
}

int solve_inverses(SolveCache* sc, const SolveFactor& f, bool lower) {
    cudaStream_t s = f.g.comm->stream;
    const int v = f.g.v, nb = f.g.nb;
    sc->inv.reset();
    int nown = 0;
    for (int t = 0; t < f.g.Nt; ++t) nown += diag_slot(f, t) >= 0;
    const size_t per = 2 * (size_t)v * nb;
    CFLX_TRY(sc->inv.alloc(std::max(1, nown) * per));
    DevBuf<double> tile, linvT;
    CFLX_TRY(tile.alloc((size_t)v * v));
    CFLX_TRY(linvT.alloc((size_t)v * nb));
    int rc = CFLX_OK;
    for (int t = 0; t < f.g.Nt && !rc; ++t) {
        const int slot = diag_slot(f, t);
        if (slot < 0) continue;
        rc = solve_tile_inverses(diag_tile(f, t), f.g.Nl, v, nb, lower, sc->inv + slot * per, tile, linvT, s);
    }
    if (cudaStreamSynchronize(s) != cudaSuccess && !rc) rc = CFLX_ERR_CUDA;
    return rc;
}

int solve_set_rows(DevBuf<int>* dst, const std::vector<int>& rows, cudaStream_t s) {
    if (!*dst) CFLX_TRY(dst->alloc(rows.size()));
    CFLX_CUDA(cudaMemcpyAsync(*dst, rows.data(), sizeof(int) * rows.size(), cudaMemcpyHostToDevice, s));
    CFLX_CUDA(cudaStreamSynchronize(s));  // `rows` is a host temporary
    return CFLX_OK;
}

// Z[r][j] *= sgn[global column of local column r], for the local columns of real tiles (global index < M); a
// grid-stride loop over the Nl x ldn entries
__global__ void solve_signs_kernel(double* __restrict__ Z, int ldn, Layout L, const double* __restrict__ sgn) {
    const int64_t n = (int64_t)L.Nl * ldn;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
        const int gc = L.col((int)(e / ldn));
        if (gc < L.M) Z[e] *= sgn[gc];
    }
}

int solve_seed(SolveCache* sc, const SolveFactor& f, int ldn, int nrhs, const double* B, int ldb, const SolveSeed& at) {
    cudaStream_t s = f.g.comm->stream;
    CFLX_CUDA(cudaMemsetAsync(sc->X, 0, sizeof(double) * f.g.M * ldn, s));
    if (sc->W) CFLX_CUDA(cudaMemsetAsync(sc->W, 0, sizeof(double) * f.g.Ml * ldn, s));
    if (sc->Z) CFLX_CUDA(cudaMemsetAsync(sc->Z, 0, sizeof(double) * f.g.Nl * ldn, s));
    const bool holds = f.g.pk == 0 && (at.by_col ? f.g.pi : f.g.pj) == 0;
    if (holds && at.n > 0) {
        CFLX_CUDA(cudaMemsetAsync(sc->B, 0, sizeof(double) * f.g.M * ldn, s));
        CFLX_CUDA(cudaMemcpy2DAsync(sc->B, ldn * sizeof(double), B, (size_t)ldb * sizeof(double), nrhs * sizeof(double),
                                    f.g.M, cudaMemcpyDefault, s));
        CFLX_TRY(launch_gather_rows(sc->B, ldn, at.rows, at.n, ldn, at.dst, s));
    }
    return CFLX_OK;
}

int solve_row_sweep(SolveCache* sc, const SolveFactor& f, int ldn, bool forward, double* keep, int keep_div,
                    bool clear_row, int t_lo, int t_hi) {
    cudaStream_t s = f.g.comm->stream;
    const int v = f.g.v, Px = f.g.Px, Py = f.g.Py, Nl = f.g.Nl, tiles = f.rows / v;
    const bool layer0 = f.g.pk == 0;
    const size_t tile = (size_t)v * ldn;
    if (t_hi < 0) t_hi = f.g.Nt;
    for (int i = t_lo; i < t_hi; ++i) {
        const int t = forward ? i : t_lo + t_hi - 1 - i;
        const bool in_row = f.g.pi == t % Px, in_col = f.g.pj == t % Py, owner = layer0 && in_row && in_col;
        double* const Wt = sc->W + (int64_t)(t / Px) * tile;
        double* R = Wt;  // tile t's rows of W, summed over the grid row onto the diagonal owner
        if (in_row && Py * f.stride > 1) {
            CFLX_NCCL(ncclReduce(Wt, sc->R, tile, ncclDouble, ncclSum, (t % Py) * f.stride, f.row_comm->c, s));
            R = sc->R;
        }
        if (owner) {
            CFLX_TRY(diag_solve_tile(*sc, f, t, forward ? Tri::Lower : Tri::Upper, R, ldn, s));
            CFLX_CUDA(cudaMemcpyAsync(keep + (int64_t)(t / keep_div) * tile, sc->Y, tile * sizeof(double),
                                      cudaMemcpyDeviceToDevice, s));
        } else if (clear_row && in_row && layer0) {
            CFLX_CUDA(cudaMemsetAsync(Wt, 0, tile * sizeof(double), s));
        }
        if (in_col && Px * f.stride > 1)
            CFLX_NCCL(ncclBroadcast(sc->Y, sc->Y, tile, ncclDouble, (t % Px) * f.stride, f.col_comm->c, s));
        // W[tiles I > t] -= L[I, t] Y_t (forward), W[tiles I < t] -= U[I, t] X_t (backward), on the grid column
        const int lo = forward ? std::min(tiles, first_local_tile(t + 1, f.g.pi, Px)) * v : 0;
        const int hi = forward ? f.rows : std::min(tiles, first_local_tile(t, f.g.pi, Px)) * v;
        if (in_col && layer0 && lo < hi)
            CFLX_TRY(launch_gemm_narrow(hi - lo, ldn, v, f.F + (int64_t)lo * Nl + (int64_t)(t / Py) * v, Nl, sc->Y, ldn,
                                        sc->W + (int64_t)lo * ldn, ldn, sc->W + (int64_t)lo * ldn, ldn, -1.0, 1.0, s));
    }
    return CFLX_OK;
}

int solve_col_sweep(SolveCache* sc, const SolveFactor& f, int ldn, bool forward, Tri tri, double* keep, int keep_div,
                    bool clear_col, int t_lo, int t_hi) {
    cudaStream_t s = f.g.comm->stream;
    const int v = f.g.v, Px = f.g.Px, Py = f.g.Py, Nl = f.g.Nl;
    const bool layer0 = f.g.pk == 0;
    const size_t tile = (size_t)v * ldn;
    if (t_hi < 0) t_hi = f.g.Nt;
    const int c_lo = first_local_tile(t_lo, f.g.pj, Py) * v;  // local columns with gj < t_lo are never updated
    for (int i = t_lo; i < t_hi; ++i) {
        const int t = forward ? i : t_lo + t_hi - 1 - i;
        const bool in_row = f.g.pi == t % Px, in_col = f.g.pj == t % Py, owner = layer0 && in_row && in_col;
        double* const Zt = sc->Z + (int64_t)(t / Py) * tile;
        double* R = Zt;  // tile t's columns of Z, summed over the grid column onto the owner
        if (in_col && Px * f.stride > 1) {
            CFLX_NCCL(ncclReduce(Zt, sc->R, tile, ncclDouble, ncclSum, (t % Px) * f.stride, f.col_comm->c, s));
            R = sc->R;
        }
        if (owner) {
            CFLX_TRY(diag_solve_tile(*sc, f, t, tri, R, ldn, s));
            CFLX_CUDA(cudaMemcpyAsync(keep + (int64_t)(t / keep_div) * tile, sc->Y, tile * sizeof(double),
                                      cudaMemcpyDeviceToDevice, s));
        } else if (clear_col && in_col && layer0) {
            CFLX_CUDA(cudaMemsetAsync(Zt, 0, tile * sizeof(double), s));
        }
        if (!in_row) continue;
        if (Py * f.stride > 1)
            CFLX_NCCL(ncclBroadcast(sc->Y, sc->Y, tile, ncclDouble, (t % Py) * f.stride, f.row_comm->c, s));
        if (!layer0) continue;
        const double* Ft = f.F + (int64_t)(t / Px) * v * Nl;  // local tile row t / Px
        if (forward) {  // Z[columns gj > t] -= U[t, gj]^T Y_t: a suffix of the tile row
            const int lo = first_local_tile(t + 1, f.g.pj, Py) * v;
            if (lo < Nl)
                CFLX_TRY(launch_gemm_narrow_tn(Nl - lo, ldn, v, Ft + lo, Nl, sc->Y, ldn, sc->Z + (int64_t)lo * ldn, ldn,
                                               sc->Z + (int64_t)lo * ldn, ldn, -1.0, 1.0, s));
        } else {
            const int m = first_local_tile(t, f.g.pj, Py) * v;  // local columns with gj < t: a prefix of the tile row
            if (m > c_lo)  // Z[columns t_lo <= gj < t] -= L[t, gj]^T X_t
                CFLX_TRY(launch_gemm_narrow_tn(m - c_lo, ldn, v, Ft + c_lo, Nl, sc->Y, ldn, sc->Z + (int64_t)c_lo * ldn, ldn,
                                               sc->Z + (int64_t)c_lo * ldn, ldn, -1.0, 1.0, s));
        }
    }
    return CFLX_OK;
}

int solve_apply_signs(SolveCache* sc, const SolveFactor& f, int ldn) {
    if (!f.sgn || f.g.pk != 0) return CFLX_OK;
    return launch_solve_signs(sc->Z, ldn, f.g, f.sgn, f.g.comm->stream);
}

int launch_solve_signs(double* Z, int ldn, const Layout& L, const double* sgn, cudaStream_t s) {
    const int64_t n = (int64_t)L.Nl * ldn;
    if (n <= 0) return CFLX_OK;
    solve_signs_kernel<<<(unsigned)std::min<int64_t>((n + 255) / 256, 4096), 256, 0, s>>>(Z, ldn, L, sgn);
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}

int solve_finish(SolveCache* sc, const SolveFactor& f, int ldn, int nrhs, double* X, int ldx, const int* unperm) {
    cudaStream_t s = f.g.comm->stream;
    // exactly one rank contributes each element: the sum is X itself, bit for bit, on every rank
    if (f.g.P > 1) CFLX_NCCL(ncclAllReduce(sc->X, sc->X, (size_t)f.g.M * ldn, ncclDouble, ncclSum, f.g.comm->world, s));
    const double* out = sc->X;
    if (unperm) {
        CFLX_TRY(launch_gather_rows(sc->X, ldn, unperm, f.g.M, ldn, sc->Xg, s));
        out = sc->Xg;
    }
    if (X)
        CFLX_CUDA(cudaMemcpy2DAsync(X, (size_t)ldx * sizeof(double), out, ldn * sizeof(double), nrhs * sizeof(double),
                                    f.g.M, cudaMemcpyDefault, s));
    CFLX_CUDA(cudaStreamSynchronize(s));
    return CFLX_OK;
}

// ---------------------------------------------------------------- the 1-norm condition estimate
// LAPACK's dlacn2 (Lacn2, refine.cu) driven to the end: kase 1 asks for inv(A) x, kase 2 for inv(A)^T x.
int estimate_inv_norm1(int n, const std::function<int(int, double*)>& apply, double* est_out) {
    Lacn2 st;
    st.start(n);
    while (st.kase != 0) {
        CFLX_TRY(apply(st.kase, st.x.data()));
        st.step();
    }
    *est_out = st.est;
    return CFLX_OK;
}

double rcond_from(double anorm, double ainvnm) {
    if (!(anorm > 0.0) || !(ainvnm > 0.0) || !std::isfinite(ainvnm)) return 0.0;
    const double r = (1.0 / ainvnm) / anorm;
    return std::isfinite(r) ? r : 0.0;
}

}  // namespace cflx
