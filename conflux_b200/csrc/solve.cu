// conflux_b200/csrc/solve.cu -- A X = B with the factors of the last cflx_lu_factor (P A = L U), on the GPU grid.
//
// The factors are first brought into the conflux block-cyclic layout of the validation path (redistribute_pivoted_rows,
// validate.cu): tile (I, J) of L\U on rank (I % Px, J % Py, 0).  The solve is then a forward and a backward sweep over
// the tile diagonal.  Every rank keeps a partial right-hand side W (Ml x ldn, its tile rows); the sum of W over a grid
// row is the current right-hand side of those tile rows.  Step t of a sweep:
//   ncclReduce of tile t's rows of W over the grid row (jk-communicator) onto the diagonal owner (t % Px, t % Py, 0);
//   the owner solves with L_tt (U_tt) by an nb-block sweep with the inverses of the nb x nb diagonal blocks;
//   ncclBroadcast of the solved tile over the grid column (ik-communicator);
//   every layer-0 rank of that grid column subtracts L[I, t] * Y_t (U[I, t] * X_t) from its rows of the tiles I > t
//   (I < t).
// The diagonal owners write X_t into a zeroed M x ldn buffer, and one all-reduce makes X identical on every rank.  All
// arithmetic is gemm_narrow_kernel: a factor block (row-major, read in place) times a few right-hand sides.
#include <cstring>

#include "lu_state.h"

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
constexpr int NW = 4;         // warps per CTA
constexpr int BM = 16 * NW;   // rows per CTA
constexpr int KC = 64;        // k rows per chunk (B in shared memory, A in registers)

struct NarrowArgs {
    int M, N, K;
    const double* A;
    int64_t lda;
    const double* B;
    int64_t ldb;
    const double* C;  // read only when beta != 0; may alias D
    int64_t ldc;
    double* D;
    int64_t ldd;
    double alpha, beta;
};

__device__ __forceinline__ void cp_async8(double* smem, const double* gmem, bool valid) {  // zero-fills when !valid
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;" ::"r"(smem_u32(smem)), "l"(gmem), "r"(valid ? 8 : 0)
                 : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

// k-pair rows of BN + 1 double2: the 8 lanes of a quarter warp (g = 0, 1; t = 0..3) read k pairs 2t + h, and
// 2t * (BN + 1) + g covers 8 distinct 16-byte bank groups
template <int NT>
struct NarrowCfg {
    static constexpr int BN = 8 * NT, LDP = BN + 1;
    static constexpr size_t STAGE = (size_t)KC / 2 * LDP;  // double2 per buffer
    static constexpr size_t SMEM = 2 * STAGE * sizeof(double2);
};

// B rows [kc, kc + KC) x columns [n0, n0 + BN) of chunk kc into one buffer, as k pairs
template <int NT>
__device__ __forceinline__ void stage_b(const NarrowArgs& g, int kc, int n0, double2* buf) {
    constexpr int BN = NarrowCfg<NT>::BN, LDP = NarrowCfg<NT>::LDP;
    double* d = reinterpret_cast<double*>(buf);
    for (int e = threadIdx.x; e < KC * BN; e += NW * 32) {
        const int kk = e / BN, n = e % BN, k = kc + kk, col = n0 + n;
        const bool ok = k < g.K && col < g.N;
        cp_async8(d + 2 * ((kk >> 1) * LDP + n) + (kk & 1), ok ? g.B + (int64_t)k * g.ldb + col : g.B, ok);
    }
    cp_async_commit();
}

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
    if (cfg.raise(C::SMEM))
        CFLX_CUDA(cudaFuncSetAttribute(gemm_narrow_kernel<NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM));
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
    if (cfg.raise(C::SMEM))
        CFLX_CUDA(cudaFuncSetAttribute(gemm_narrow_tn_kernel<NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM));
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

int launch_transpose_blocks(const double* in, int nb, int64_t total, double* out, cudaStream_t stream) {
    transpose_blocks_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(in, nb, total, out);
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}

namespace {
// ---------------------------------------------------------------- solve
// slot of diagonal tile t in sv_inv on this rank (-1: not owned)
int diag_slot(const cflx_lu* lu, int t) {
    if (lu->pk != 0 || t % lu->Px != lu->pi || t % lu->Py != lu->pj) return -1;
    int n = 0;
    for (int u = 0; u < t; ++u) n += (u % lu->Px == lu->pi && u % lu->Py == lu->pj);
    return n;
}

// First call after a factorisation: factors in the conflux layout (Cbuf, as cflx_lu_get_factors leaves them), the
// inverses of the nb x nb diagonal blocks of every owned diagonal tile (Linv row-major, then Uinv), and on the ranks
// that seed the right-hand side, the row of B that each local row of P*B comes from.
int solve_prepare(cflx_lu* lu) {
    cflx_comm* c = lu->comm;
    cudaStream_t s = c->stream;
    const int v = lu->v, nb = lu->nb, Px = lu->Px, Py = lu->Py, Ml = lu->Ml, Nl = lu->Nl;
    std::vector<int> hist(lu->M);
    CFLX_TRY(cflx_lu_get_permutation(lu, hist.data()));
    cudaFree(lu->sv_inv);
    lu->sv_inv = nullptr;
    if (lu->pk == 0) {
        if (!lu->Cbuf) CFLX_TRY(dmalloc(&lu->Cbuf, (size_t)Ml * Nl));
        int rc = redistribute_pivoted_rows(lu, hist, true, lu->A11, lu->Cbuf);
        cudaFree(lu->xbuf);  // 2 x local matrix of staging: do not keep it alive
        lu->xbuf = nullptr;
        if (rc) return rc;
        int nown = 0;
        for (int t = 0; t < lu->Nt; ++t) nown += diag_slot(lu, t) >= 0;
        const size_t per = 2 * (size_t)v * nb;
        CFLX_TRY(dmalloc(&lu->sv_inv, std::max(1, nown) * per));
        double *tile = nullptr, *linvT = nullptr;
        rc = dmalloc(&tile, (size_t)v * v);
        if (!rc) rc = dmalloc(&linvT, (size_t)v * nb);
        for (int t = 0; t < lu->Nt && !rc; ++t) {
            const int slot = diag_slot(lu, t);
            if (slot < 0) continue;
            double* inv = lu->sv_inv + slot * per;
            const double* ctt = lu->Cbuf + (int64_t)(t / Px) * v * Nl + (int64_t)(t / Py) * v;
            if (cudaMemcpy2DAsync(tile, v * sizeof(double), ctt, Nl * sizeof(double), v * sizeof(double), v,
                                  cudaMemcpyDeviceToDevice, s) != cudaSuccess) {
                set_last_error("solve: diagonal tile copy failed");
                rc = CFLX_ERR_CUDA;
                break;
            }
            rc = launch_diag_inverses(tile, v, nb, inv + (size_t)v * nb, linvT, s);
            if (!rc) rc = launch_transpose_blocks(linvT, nb, (int64_t)v * nb, inv, s);
        }
        if (cudaStreamSynchronize(s) != cudaSuccess && !rc) rc = CFLX_ERR_CUDA;
        cudaFree(tile);
        cudaFree(linvT);
        if (rc) return rc;
        if (lu->pj == 0) {  // local row (k / Px)*v + i of P*B is row hist[k*v + i] of B, for the tiles k of this grid row
            std::vector<int> rows(Ml, 0);
            for (int q = 0; q < lu->M; ++q) {
                const int k = q / v;
                if (k % Px == lu->pi) rows[(k / Px) * v + q % v] = hist[q];
            }
            if (!lu->sv_rows) CFLX_TRY(dmalloc(&lu->sv_rows, (size_t)Ml));
            CFLX_CUDA(cudaMemcpyAsync(lu->sv_rows, rows.data(), sizeof(int) * Ml, cudaMemcpyHostToDevice, s));
            CFLX_CUDA(cudaStreamSynchronize(s));  // `rows` is a host temporary
        }
    }
    lu->solve_ready = true;
    return CFLX_OK;
}

int ensure_solve_buffers(cflx_lu* lu, int ldn) {
    if (ldn <= lu->sv_ldn) return CFLX_OK;
    for (double** p : {&lu->sv_B, &lu->sv_W, &lu->sv_R, &lu->sv_Y, &lu->sv_X}) {
        cudaFree(*p);
        *p = nullptr;
    }
    lu->sv_ldn = 0;
    const size_t M = lu->M, Ml = lu->Ml, v = lu->v;
    if (lu->pk == 0 && lu->pj == 0) CFLX_TRY(dmalloc(&lu->sv_B, M * ldn));
    CFLX_TRY(dmalloc(&lu->sv_W, Ml * ldn));
    CFLX_TRY(dmalloc(&lu->sv_R, v * ldn));
    CFLX_TRY(dmalloc(&lu->sv_Y, v * ldn));
    CFLX_TRY(dmalloc(&lu->sv_X, M * ldn));
    lu->sv_ldn = ldn;
    return CFLX_OK;
}

// Y = L_tt^-1 R (forward) or Y = U_tt^-1 R (backward) on the diagonal owner; R (v x ldn) is overwritten
int diag_solve(cflx_lu* lu, int t, bool lower, double* R, double* Y, int ldn, cudaStream_t s) {
    const int v = lu->v, nb = lu->nb, Nl = lu->Nl, nblk = v / nb;
    const double* inv = lu->sv_inv + diag_slot(lu, t) * 2 * (size_t)v * nb + (lower ? 0 : (size_t)v * nb);
    const double* ctt = lu->Cbuf + (int64_t)(t / lu->Px) * v * Nl + (int64_t)(t / lu->Py) * v;
    for (int i = 0; i < nblk; ++i) {
        const int j = lower ? i : nblk - 1 - i;
        const int64_t o = (int64_t)j * nb * ldn;
        CFLX_TRY(launch_gemm_narrow(nb, ldn, nb, inv + (size_t)j * nb * nb, nb, R + o, ldn, nullptr, ldn, Y + o, ldn, 1.0,
                                    0.0, s));
        if (lower && j + 1 < nblk) {  // R_i -= L_ij Y_j, i > j
            const int64_t o1 = (int64_t)(j + 1) * nb;
            CFLX_TRY(launch_gemm_narrow(v - (j + 1) * nb, ldn, nb, ctt + o1 * Nl + (int64_t)j * nb, Nl, Y + o, ldn,
                                        R + o1 * ldn, ldn, R + o1 * ldn, ldn, -1.0, 1.0, s));
        }
        if (!lower && j > 0)  // R_i -= U_ij X_j, i < j
            CFLX_TRY(launch_gemm_narrow(j * nb, ldn, nb, ctt + (int64_t)j * nb, Nl, Y + o, ldn, R, ldn, R, ldn, -1.0, 1.0, s));
    }
    return CFLX_OK;
}
}  // namespace

int lu_solve_grid(cflx_lu* lu, int nrhs, const double* B, int ldb, double* X, int ldx) {
    cflx_comm* c = lu->comm;
    cudaStream_t s = c->stream;
    if (!lu->solve_ready) CFLX_TRY(solve_prepare(lu));
    const int v = lu->v, Px = lu->Px, Py = lu->Py, Pz = lu->Pz, Ml = lu->Ml, Nl = lu->Nl, Nt = lu->Nt, M = lu->M;
    const int pi = lu->pi, pj = lu->pj;
    const bool layer0 = lu->pk == 0;
    const int ldn = (int)round_up(nrhs, 8);
    CFLX_TRY(ensure_solve_buffers(lu, ldn));
    double *W = lu->sv_W, *Y = lu->sv_Y, *Xd = lu->sv_X;
    const size_t tile = (size_t)v * ldn;
    CFLX_CUDA(cudaMemsetAsync(W, 0, sizeof(double) * Ml * ldn, s));
    CFLX_CUDA(cudaMemsetAsync(Xd, 0, sizeof(double) * M * ldn, s));
    // W = rows of P*B on the first grid column, 0 elsewhere
    if (layer0 && pj == 0) {
        CFLX_CUDA(cudaMemsetAsync(lu->sv_B, 0, sizeof(double) * M * ldn, s));
        CFLX_CUDA(cudaMemcpy2DAsync(lu->sv_B, ldn * sizeof(double), B, (size_t)ldb * sizeof(double), nrhs * sizeof(double), M,
                                    cudaMemcpyHostToDevice, s));
        CFLX_TRY(launch_gather_rows(lu->sv_B, ldn, lu->sv_rows, Ml, ldn, W, s));
    }
    auto first_local_tile = [&](int t) { return std::min(Ml / v, (t - pi + Px - 1) / Px); };  // first local tile >= t
    // tile t's rows of W, summed over the grid row, onto the diagonal owner; returns where the sum is
    auto reduce_tile = [&](int t, double** R) -> int {
        *R = W + (int64_t)(t / Px) * tile;
        if (Py * Pz > 1) {
            CFLX_NCCL(ncclReduce(*R, lu->sv_R, tile, ncclDouble, ncclSum, (t % Py) * Pz, lu->jk_comm.c, s));
            *R = lu->sv_R;
        }
        return CFLX_OK;
    };
    auto bcast_tile = [&](int t) -> int {
        if (Px * Pz > 1) CFLX_NCCL(ncclBroadcast(Y, Y, tile, ncclDouble, (t % Px) * Pz, lu->ik_comm.c, s));
        return CFLX_OK;
    };
    // ---- forward sweep: L Y = P B
    for (int t = 0; t < Nt; ++t) {
        const bool in_row = pi == t % Px, in_col = pj == t % Py, owner = layer0 && in_row && in_col;
        double* R = nullptr;
        if (in_row) CFLX_TRY(reduce_tile(t, &R));
        if (owner) CFLX_TRY(diag_solve(lu, t, true, R, Y, ldn, s));
        if (in_col) CFLX_TRY(bcast_tile(t));
        if (in_row && layer0) {  // the backward sweep starts from W = Y, held by the diagonal owners
            double* Wt = W + (int64_t)(t / Px) * tile;
            if (owner) CFLX_CUDA(cudaMemcpyAsync(Wt, Y, tile * sizeof(double), cudaMemcpyDeviceToDevice, s));
            else CFLX_CUDA(cudaMemsetAsync(Wt, 0, tile * sizeof(double), s));
        }
        const int row_lo = first_local_tile(t + 1) * v;
        if (in_col && layer0 && row_lo < Ml) {  // W[tiles I > t] -= L[I, t] Y_t
            CFLX_TRY(launch_gemm_narrow(Ml - row_lo, ldn, v, lu->Cbuf + (int64_t)row_lo * Nl + (int64_t)(t / Py) * v, Nl, Y,
                                        ldn, W + (int64_t)row_lo * ldn, ldn, W + (int64_t)row_lo * ldn, ldn, -1.0, 1.0, s));
        }
    }
    // ---- backward sweep: U X = Y
    for (int t = Nt - 1; t >= 0; --t) {
        const bool in_row = pi == t % Px, in_col = pj == t % Py, owner = layer0 && in_row && in_col;
        double* R = nullptr;
        if (in_row) CFLX_TRY(reduce_tile(t, &R));
        if (owner) {
            CFLX_TRY(diag_solve(lu, t, false, R, Y, ldn, s));
            CFLX_CUDA(cudaMemcpyAsync(Xd + (int64_t)t * tile, Y, tile * sizeof(double), cudaMemcpyDeviceToDevice, s));
        }
        if (in_col) CFLX_TRY(bcast_tile(t));
        const int row_hi = first_local_tile(t) * v;
        if (in_col && layer0 && row_hi > 0) {  // W[tiles I < t] -= U[I, t] X_t
            CFLX_TRY(launch_gemm_narrow(row_hi, ldn, v, lu->Cbuf + (int64_t)(t / Py) * v, Nl, Y, ldn, W, ldn, W, ldn, -1.0,
                                        1.0, s));
        }
    }
    // exactly one rank contributes each element: the sum is X itself, bit for bit, on every rank
    if (lu->P > 1) CFLX_NCCL(ncclAllReduce(Xd, Xd, (size_t)M * ldn, ncclDouble, ncclSum, c->world, s));
    if (X)
        CFLX_CUDA(cudaMemcpy2DAsync(X, (size_t)ldx * sizeof(double), Xd, ldn * sizeof(double), nrhs * sizeof(double), M,
                                    cudaMemcpyDeviceToHost, s));
    CFLX_CUDA(cudaStreamSynchronize(s));
    return CFLX_OK;
}

}  // namespace cflx
