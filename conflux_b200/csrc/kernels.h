// conflux_b200/csrc/kernels.h -- host-callable launchers of the sm_90a kernels (internal; the public boundary is
// include/conflux_b200.h).
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <functional>
#include <memory>

#include "common.cuh"

namespace cflx {

// ---------------------------------------------------------------- gemm.cu
struct GemmArgs {
    int M, N, K;
    const double* AT;  // [K][ldat]  (A transposed: AT[k][m])
    int64_t ldat;
    const double* B;  // [K][ldb]
    int64_t ldb;
    const double* C;  // [M][ldc]   (read only when beta != 0)
    int64_t ldc;
    double* D;  // [M][ldd]   (may alias C)
    int64_t ldd;
    double alpha, beta;
};
int gemm_tn_setup();
int launch_gemm_tn(const GemmArgs& g, cudaStream_t stream);

// ---------------------------------------------------------------- ozaki.cu, tf32.cu: the split updates
// What the workspaces of the wgmma updates share: the per-row power-of-two exponents of both operands (cap_a / cap_b
// rows, whole CTA tiles of bm / bn rows), the contraction length and the SM count their persistent grids are capped at.
struct SplitWorkspace {
    DevBuf<int> ea;  // [cap_a]
    DevBuf<int> eb;  // [cap_b]
    int K = 0, cap_a = 0, cap_b = 0, sms = 0;
    int init(int max_rows, int max_cols, int k, int bm, int bn) {
        K = k;
        cap_a = (int)round_up(max_rows > 1 ? max_rows : 1, bm);
        cap_b = (int)round_up(max_cols > 1 ? max_cols : 1, bn);
        CFLX_TRY(ea.alloc_exact(cap_a));
        CFLX_TRY(eb.alloc_exact(cap_b));
        CFLX_CUDA(cudaMemset(ea, 0, sizeof(int) * cap_a));
        CFLX_CUDA(cudaMemset(eb, 0, sizeof(int) * cap_b));
        int dev = 0;
        CFLX_CUDA(cudaGetDevice(&dev));
        CFLX_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
        return CFLX_OK;
    }
    // CTAs of a persistent launch over `tiles` tiles: at most one per SM, and at most max_ctas when it is > 0
    int grid(int tiles, int max_ctas) const {
        const int cap = max_ctas > 0 && max_ctas < sms ? max_ctas : sms;
        return tiles < cap ? tiles : cap;
    }
};

// FP64 trailing update on the int8 wgmma path (error-free digit planes): C -= L * U with L^T, U K-major in HBM.
struct OzakiWorkspace : SplitWorkspace {
    struct Maps;                // the two CUtensorMap objects (kept out of this header)
    DevBuf<int8_t> planesA;     // [8][cap_a][K]
    DevBuf<int8_t> planesB;     // [8][cap_b][K]
    std::unique_ptr<Maps> maps;
    OzakiWorkspace();
    ~OzakiWorkspace();  // where Maps is complete
};
// on a new workspace
int ozaki_workspace_create(OzakiWorkspace* ws, int max_rows, int max_cols, int K);
int ozaki_split_a(OzakiWorkspace* ws, const double* LT, int64_t ld, int n, cudaStream_t s);
int ozaki_split_b(OzakiWorkspace* ws, const double* U, int64_t ld, int col0, int n, cudaStream_t s);
int wgmma_peak_probe(int n, double* tmacs_out);
int launch_ozaki_gemm(OzakiWorkspace* ws, int M, int N, int row0, int col0, double* C, int64_t ldc, int max_ctas, cudaStream_t s);

// The low-precision trailing update of the mixed-precision drivers on the TF32 wgmma path: C -= L * U with L^T, U K-major
// in HBM, split into per-row power-of-two scaled TF32 terms (hi, and lo for terms = 3), FP32 accumulation, FP64 C.
struct Tf32Workspace : SplitWorkspace {
    struct Maps;               // the four CUtensorMap objects (kept out of this header)
    DevBuf<float> hiA, loA;    // [cap_a][KP]
    DevBuf<float> hiB, loB;    // [cap_b][KP]
    std::unique_ptr<Maps> maps;
    int KP = 0;  // K rounded up to 8 (the tail is zero)
    Tf32Workspace();
    ~Tf32Workspace();  // where Maps is complete
};
// on a new workspace; any K >= 1
int tf32_workspace_create(Tf32Workspace* ws, int max_rows, int max_cols, int K);
// terms 1 or 3 (3 also writes the lo slabs)
int tf32_split_a(Tf32Workspace* ws, int terms, const double* LT, int64_t ld, int n, cudaStream_t s);
int tf32_split_b(Tf32Workspace* ws, int terms, const double* U, int64_t ld, int col0, int n, cudaStream_t s);
// launch_ozaki_gemm's window; ldc even, C 16-byte aligned, any M, N >= 1
int launch_tf32_gemm(Tf32Workspace* ws, int terms, int M, int N, int row0, int col0, double* C, int64_t ldc, int max_ctas,
                     cudaStream_t s);

// ---------------------------------------------------------------- update.cu
// The trailing update C -= L U of a factorisation.  Its kind is fixed at creation: the FP64 DMMA kernel (gemm.cu), or
// the int8 digit planes (ozaki.cu); a TF32 or TF32x3 kind (tf32.cu) takes over for the factorisations of one
// mixed-precision driver (with_tf32).  The split kinds run a persistent kernel on operands split beforehand: split_a /
// split_b fill them (no-ops for FP64, see splits()), apply reads a window of them.
struct TrailingUpdate {
    OzakiWorkspace oz;  // the int8 kind's digit planes
    Tf32Workspace tf;   // the TF32 terms, made by the first with_tf32
    int rows = 0, cols = 0, K = 0;
    bool int8 = false;
    int terms = 0;  // with_tf32's kind while it runs: 1 (TF32) or 3 (TF32x3); 0 otherwise

    // operands of up to rows of L^T and cols of U with contraction length K; the int8 kind when `int8`, else FP64
    int create(int rows, int cols, int K, bool int8);
    // fn() on the TF32 kind of `terms` (1 or 3) terms; the kind of create again on return
    int with_tf32(int terms, const std::function<int()>& fn);
    // a persistent split kernel runs: split_a / split_b launch their kernel (callers count the launches by this)
    bool splits() const { return int8 || terms; }
    // the TF32 kind runs (the factors are not those of an FP64 update)
    bool tf32() const { return terms != 0; }
    // rows [0, n) of L^T (AT[k][row], ld) -> the A operand
    int split_a(const double* AT, int64_t ld, int n, cudaStream_t s);
    // columns [col0, col0 + n) of U (B[k][col], ld) -> the B operand, rows col0 ..
    int split_b(const double* B, int64_t ld, int col0, int n, cudaStream_t s);
    // The FP64 kind: launch_gemm_tn(g).  A split kind: g.D (g.M x g.N, g.ldd) -= A operand rows row0 .. times B operand
    // rows col0 .., on all SMs but leave_sms (when > 0).
    int apply(const GemmArgs& g, int row0, int col0, int leave_sms, cudaStream_t s);
};

// ---------------------------------------------------------------- panel.cu
// Partial-pivot LU of the n x v panel stored TRANSPOSED in W (W[c][r], ld = ldw), in place, rows never move:
// afterwards W[:, r] holds row r of L\U (multipliers left of its pivot column, U from it on, for pivot rows;
// multipliers only for the others).  perm_out[0..v) = LAPACK-equivalent winners (row index chosen at step j,
// identity beyond min(n, v)); see panel.cu for the tie-breaking contract.
struct PanelWorkspace {
    DevBuf<uint2> slot_hdr;   // [2][132][4]  LL words (payload32, epoch)
    DevBuf<uint2> slot_rows;  // [2][132][64] LL words
    int epoch;          // host-side running epoch (monotonic across launches)
    int max_ctas;       // co-resident CTA budget (<= 132)
    int cta_cap;        // optional cap on the grid (look-ahead: leave SMs to the trailing update); 0 = none
    // column-owner kernel for panels of <= 1024 rows (tournament stacks)
    DevBuf<unsigned> sk_flags;   // [1024] epoch of the last publication of column block b
    DevBuf<int> sk_ppos;         // [v] LAPACK position of every pivot when it was chosen
    DevBuf<unsigned> sk_ticket;  // logical CTA ids in start order
    unsigned sk_epoch, sk_ticket_count;
    int sk_enabled;
};
// on a new workspace
int panel_workspace_create(PanelWorkspace* ws);
int launch_panel_getrf(double* W, int64_t ldw, int n, int v, int* perm_out, PanelWorkspace* ws, cudaStream_t stream);
// same, and CTA 0 also emits into A00 (v x v) the columns >= (i / nb) * nb of pivot i's L\U row; *nb_used = nb
int launch_panel_getrf_a00(double* W, int64_t ldw, int n, int v, int* perm_out, double* A00, int* nb_used,
                           PanelWorkspace* ws, cudaStream_t stream);

// ---------------------------------------------------------------- rows.cu
// PT[c][r] = A[(row0 + r) * lda + col0 + c]  for r < n, c < v     (transposing strided copy, K8/a3)
int launch_extract_panel_T(const double* A, int64_t lda, int64_t row0, int64_t col0, int n, int v, double* PT,
                           int64_t ldp, cudaStream_t stream);
// A[(row0 + r) * lda + col0 + c] = LT[c][r]                        (L written back in place)
int launch_store_panel_T(double* A, int64_t lda, int64_t row0, int64_t col0, int n, int v, const double* LT,
                         int64_t ldp, cudaStream_t stream);
// winners of a pivot search: out_vals[c][dst0 + i] = PT[c][perm[i]] (0 when perm[i] >= n_valid),
// out_tags[dst0 + i] = tags[perm[i]] (0 when padded)               (inverse_permute_rows, utils.hpp:85-116)
int launch_gather_winners(const double* PT, int64_t ldp, const int* tags, int n_valid, const int* perm, int v,
                          double* out_vals, int64_t ldo, int* out_tags, int dst0, cudaStream_t stream);
// A00[i][c] = W[c][perm[i]], A00T[c][i] = same                      (top v x v of the factored panel)
// (completes the L prefix c < (i / nb) * nb of the rows emitted by launch_panel_getrf_a00, and writes A00T)
int launch_gather_a00(const double* W, int64_t ldw, const int* perm, int v, int nb, double* A00, double* A00T,
                      cudaStream_t stream);

// One-CTA planner of step 2 (g2lnoTile + igri lookup + analyze_pivots, conflux_opt.cpp:74-148):
struct MovePlan {
    int* npiv;     // [1]
    int* cur_piv;  // [v] local rows of my pivots, tournament order
    int* order;    // [v] tournament position of my i-th pivot
    int* slot2piv; // [v] tournament position -> my pivot index, -1 if not mine
    int* early;    // [v]
    int* late;     // [v]
    int* nel;      // [1]
    int* rowsrc;   // [Ml] new local row -> old local row (identity outside the active range)
};
int launch_plan_moves(const int* gpivots, int v, int Px, int pi, int fnpr, int Ml, const int* igri, MovePlan plan,
                      cudaStream_t stream);
// push_pivots_up phases (conflux_opt.hpp:176-218), 128-bit row moves over columns [col_lo, ncols)
int launch_push_phase1(const double* A, int64_t lda, int ncols, int col_lo, MovePlan plan, int v, double* tmp,
                       double* a01raw, int64_t ld01, int c0, cudaStream_t stream);
int launch_push_phase2(double* A, int64_t lda, int ncols, int col_lo, MovePlan plan, int v, cudaStream_t stream);
int launch_push_phase3(double* A, int64_t lda, int ncols, int col_lo, int fnpr, MovePlan plan, int v,
                       const double* tmp, cudaStream_t stream);
// gri/igri bookkeeping after the push (conflux_opt.hpp:1083-1124)
int launch_update_gri(int* gri, int* gri_tmp, int* igri, const int* rowsrc, int fnpr, int Ml, int v, int Px,
                      cudaStream_t stream);
// PT2[c][r'] = PT[c][rowsrc[fnpr_new + r'] - fnpr_old], fnpr_new = fnpr_old + *npiv   (A10Buff push, :1067)
int launch_compact_panel(const double* PT, int64_t ldp, double* PT2, int64_t ldp2, const int* rowsrc, int fnpr_old,
                         const int* npiv, int Ml, int v, cudaStream_t stream);
// my pivot rows receive their U values / diagonal block:  A[(fnpr_old+i)*lda + c0 + c] = U[order[i]][c]
int launch_store_u_rows(double* A, int64_t lda, int fnpr_old, MovePlan plan, const double* U, int64_t ldu, int c0,
                        int ncols, int v, cudaStream_t stream);
int launch_store_diag(double* A, int64_t lda, int fnpr_old, MovePlan plan, const double* A00, int loff, int v,
                      cudaStream_t stream);
// residual helpers (validation only)
int launch_split_factors(const double* F, int64_t ldf, int n, double* LT, double* U, cudaStream_t stream);
int launch_gather_perm_rows(const double* A, int64_t lda, const int* perm, int n, double* out, cudaStream_t stream);
// *out += sum of X[i]^2, deterministic (the same rounding on every call); partials: SUMSQ_PARTIALS doubles of scratch
constexpr int SUMSQ_PARTIALS = 1184;
int launch_sumsq(const double* X, int64_t count, double* out, double* partials, cudaStream_t stream);
// *out += partials[0] + ... + partials[n - 1], added in a fixed order (the second pass of launch_sumsq)
int launch_sum_partials(const double* partials, int n, double* out, cudaStream_t stream);
// misc
int launch_fill(double* p, int64_t n, double val, cudaStream_t stream);
int launch_iota_gri(int* gri, int* igri, int Ml, int v, int Px, int pi, cudaStream_t stream);
int launch_pack_bcast(const double* A00, const int* tags, int v, double* buf, cudaStream_t stream);
int launch_unpack_bcast(const double* buf, int v, double* A00, double* A00T, int* gpivots, cudaStream_t stream);
int launch_record_pivots(const int* gpivots, int v, int* hist, int k, cudaStream_t stream);

// ---------------------------------------------------------------- trsm.cu
// inverses of the nb x nb diagonal blocks of A00 = L00\U00: Uinv[j] (row-major) and LinvT[j] (= inv(L_jj)^T)
int launch_diag_inverses(const double* A00, int v, int nb, double* Uinv, double* LinvT, cudaStream_t stream);
// LT = (PT * U00^-1)^T : PT, LT are [v][ld] transposed panels with n columns; PT is destroyed
int trsm_right_upper_T(const double* A00, const double* Uinv, int v, int nb, double* PT, double* LT, int64_t ld,
                       int n, cudaStream_t stream);
// U = L00^-1 * R : R, U are [v][ld] with n columns; R is destroyed
int trsm_left_lower_unit(const double* A00T, const double* LinvT, int v, int nb, double* R, double* U, int64_t ld,
                         int n, cudaStream_t stream);

// ---------------------------------------------------------------- chol.cu
// Cholesky of one v x v diagonal tile D (row-major, lower triangle read) in place: L in the lower triangle, zeros above,
// and L^T into UT.  Q (potrf_tile_scratch(v) doubles) selects the 128-block path for v % 128 == 0, v >= 256; Q == nullptr
// or any other v runs the one-CTA kernel (4 <= v <= 512).  A non-positive pivot at local column j sets *info = col0 + j + 1
// unless *info is already non-zero.  *launches grows by the launches the 128-block path counts.  potrf_setup(v) first.
size_t potrf_tile_scratch(int v);
int potrf_setup(int v);
// The signed Cholesky A = R S R^T of cflx_chol_factor_ldlt (chol.cu potrf_tile_kernel): the tiny rule's threshold, the
// device signs of the tile's columns (sg[c] = s_c = +-1) and the device counts cnt[4] += {replacements, positive,
// negative, zero pivots}.  R goes where L goes, S R^T where L^T goes.
struct LdltArgs {
    double tiny;
    double* sg;
    int* cnt;
};
// sa (may be null: the Cholesky): the signed factorisation of the tile
int potrf_tile(double* D, double* UT, double* Q, int* info, int col0, int v, cudaStream_t stream, int64_t* launches,
               const LdltArgs* sa = nullptr);
// one 128 x 128 block (leading dimensions ldd / ldu) on potrf128_kernel; Uc: a contiguous 128 x 128 copy of L^T
int potrf_block128(double* D, int ldd, double* UT, int ldu, double* Uc, int* info, int col0, cudaStream_t stream,
                   const LdltArgs* sa = nullptr);

// ---------------------------------------------------------------- fixed.cu (cflx_lu_factor_fixed)
// Unpivoted LU of one v x v block: Bt is the block transposed (Bt[c][i], as launch_gather_winners leaves it), A
// receives L\U row-major (unit L) and AT (may be null) its transpose; tags_out[i] = tags_in[i] (both may be null).  A
// pivot u with |u| < tiny becomes copysign(tiny, u) (+tiny for +-0).  rec (may be null): rec[0] += the replacements,
// rec[1] = col0 + 1 + the column of the first exactly zero pivot when rec[1] is 0.  blocked (getrf_nopiv_blocked(v)
// only): 128-wide block columns, the diagonal blocks on the one-CTA kernel, the rest on the TRSMs and gemm_tn;
// otherwise the one-CTA kernel on the whole block.  scratch: getrf_nopiv_scratch(v, blocked) doubles of device memory,
// or null when that is 0.  *launches grows by the kernels launched.  Deterministic.  gemm_tn_setup() first.
bool getrf_nopiv_blocked(int v);
size_t getrf_nopiv_scratch(int v, bool blocked);
int launch_getrf_nopiv_tile(const double* Bt, int v, double tiny, double* A, double* AT, const int* tags_in, int* tags_out,
                            int* rec, int col0, bool blocked, double* scratch, cudaStream_t stream, int64_t* launches);
// pos[i] = active panel position (local row - fnpr) of global row rows[i] where grid row pi owns it, else n_old
int launch_fixed_locate(const int* rows, int v, int Px, int pi, int fnpr, int n_old, const int* igri, int* pos,
                        cudaStream_t stream);
// rec[2] = rec[1], or INT_MAX when it is 0
int launch_fixed_info_operand(int* rec, cudaStream_t stream);

// ---------------------------------------------------------------- validate.cu
// out[i][c] = A[src_rows[i] * lda + c] for i < nrows, c < ncols (ncols, lda even; 16-byte aligned rows)
int launch_gather_rows(const double* A, int64_t lda, const int* src_rows, int nrows, int ncols, double* out,
                       cudaStream_t stream);

// ---------------------------------------------------------------- solve.cu
// D = beta * C + alpha * A * B: A [M x K] row-major (lda even, 16-byte aligned), B [K x N], C / D [M x N] (D may alias
// C; C is read only when beta != 0).  K % 4 == 0; any M, N >= 1.  Memory-bound on A: the narrow GEMM of the solve.
int launch_gemm_narrow(int M, int N, int K, const double* A, int64_t lda, const double* B, int64_t ldb, const double* C,
                       int64_t ldc, double* D, int64_t ldd, double alpha, double beta, cudaStream_t stream);
// D = beta * C + alpha * AT^T * B: AT [K x M] row-major, read in place (ldat even and >= M, AT 16-byte aligned), B [K x N],
// C / D [M x N] (D may alias C; C is read only when beta != 0).  Any K >= 0 and M, N >= 1; nothing beyond M, K or N is
// read.  Otherwise CFLX_ERR_UNSUPPORTED.  The backward sweep of the Cholesky solve (L^T with only L stored).
int launch_gemm_narrow_tn(int M, int N, int K, const double* AT, int64_t ldat, const double* B, int64_t ldb,
                          const double* C, int64_t ldc, double* D, int64_t ldd, double alpha, double beta,
                          cudaStream_t stream);

// ---------------------------------------------------------------- refine.cu
// what the residual kernels multiply (lu_state.h launch_residual)
enum class ResidMode { NN, TN, SymLower };

}  // namespace cflx
