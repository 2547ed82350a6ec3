// conflux_b200/csrc/lu_state.h -- internal state of a process-grid handle and of one factorisation plan, shared by the
// orchestration (lu.cu), the validation path (validate.cu), the solve engine (solve.cu) and the Cholesky path (chol.cu).
// Not part of the C ABI.
#pragma once
#include <nccl.h>

#include <algorithm>
#include <cmath>
#include <functional>
#include <vector>

#include "../../include/conflux_b200.h"
#include "common.cuh"
#include "kernels.h"

#define CFLX_NCCL(call)                                                                                    \
    do {                                                                                                   \
        ncclResult_t r__ = (call);                                                                         \
        if (r__ != ncclSuccess) {                                                                          \
            ::cflx::set_last_error("%s:%d: %s -> %s", __FILE__, __LINE__, #call, ncclGetErrorString(r__)); \
            return CFLX_ERR_NCCL;                                                                          \
        }                                                                                                  \
    } while (0)

struct cflx_comm {
    int world_size = 1, world_rank = 0, device = 0;
    ncclComm_t world = nullptr;
    cflx::Stream stream;
    cflx::DevBuf<double> d_scratch;  // 1 double for barriers
};

namespace cflx {
struct SubComm {
    ncclComm_t c = nullptr;
    int size = 1, rank = 0;
};

enum Phase { PH_PANEL = 0, PH_TOURN, PH_MOVES, PH_REDUCE, PH_TRSM, PH_GEMM, PH_STORE, PH_OTHER, PH_COUNT };

// Profiling regions, named like the reference's semiprof regions (PE(...) in conflux_opt.hpp; profiler.hpp:5-19) so
// that an Nsight Systems timeline (NVTX ranges) or cflx_lu_timeline() reads like the reference's profiler summary.
enum Region {
    RG_init = 0, RG_step0_copy, RG_step0_reduce, RG_step1_A10copy, RG_step1_lup, RG_step1_rowpermute, RG_step1_pivoting,
    RG_step1_A00Buff_bcast, RG_step2_pushingpivots, RG_step2_reduce, RG_step4_reshuffling, RG_step4_dtrsm, RG_step4_comm,
    RG_step5_dtrsm, RG_step5_comm, RG_step6_dgemm, RG_storingresults, RG_COUNT
};
inline const char* region_name(int r) {
    static const char* n[RG_COUNT] = {"init", "step0_copy", "step0_reduce", "step1_A10copy", "step1_lup", "step1_rowpermute",
                                      "step1_pivoting", "step1_A00Buff_bcast", "step2_pushingpivots", "step2_reduce",
                                      "step4_reshuffling", "step4_dtrsm", "step4_comm", "step5_dtrsm", "step5_comm",
                                      "step6_dgemm", "storingresults"};
    return n[r];
}
inline int region_phase(int r) {
    static const int p[RG_COUNT] = {PH_OTHER, PH_PANEL, PH_PANEL, PH_PANEL, PH_PANEL, PH_PANEL, PH_TOURN, PH_TOURN, PH_MOVES,
                                    PH_REDUCE, PH_MOVES, PH_TRSM, PH_REDUCE, PH_TRSM, PH_REDUCE, PH_GEMM, PH_STORE};
    return p[r];
}

int make_sub(cflx_comm* c, int color, int key, int size, SubComm* out);
int grid_barrier(cflx_comm* c);

// first local tile row (column) whose global tile index is >= g, on grid row (column) p of P
inline int first_local_tile(int g, int p, int P) { return g <= p ? 0 : (g - p + P - 1) / P; }

// A rank's share of the M x M block-cyclic matrix, as every pass over the input reads it: global tile (I, J) lives on
// grid position (I % Px, J % Py) at local tile (I / Px, J / Py) of the row-major Ml x Nl share.  Plain ints: kernels take
// it by value.
struct Layout {
    int M = 0;   // padded global order
    int v = 0;   // tile
    int Nt = 0;  // real tiles on the diagonal (the LU's Nt, the reference's Kappa on the Cholesky path)
    int Ml = 0, Nl = 0;
    int Px = 1, Py = 1, pi = 0, pj = 0;

    // global index of local index l at position p of a grid dimension of P
    __host__ __device__ static int global(int l, int P, int p, int v) { return ((l / v) * P + p) * v + l % v; }
    // the global row of local row r and the global column of local column c (I: the width of the result)
    template <class I = int>
    __host__ __device__ I row(int r) const { return ((I)(r / v) * Px + pi) * v + r % v; }
    template <class I = int>
    __host__ __device__ I col(int c) const { return ((I)(c / v) * Py + pj) * v + c % v; }
    // this share holds diagonal tile t, at local rows / columns from diag_row(t) / diag_col(t)
    __host__ __device__ bool holds_diag(int t) const {
        return t % Px == pi && t % Py == pj && diag_row(t) < Ml && diag_col(t) < Nl;
    }
    __host__ __device__ int diag_row(int t) const { return (t / Px) * v; }
    __host__ __device__ int diag_col(int t) const { return (t / Py) * v; }
};

// A handle's process grid: the layout of this rank's share, its place in the Px x Py x Pz grid (row-major numbering,
// rank = (pi * Py + pj) * Pz + pk), and the sub-communicators every handle makes.
struct Grid : Layout {
    cflx_comm* comm = nullptr;
    int Pz = 1, P = 1, pk = 0, rank = 0;
    int nlayr = 0;  // contraction indices of one z layer
    int nb = 0;     // diagonal inverse block
    SubComm k_comm, i_comm;
};
// the rank's grid position, then the k (same (pi, pj)) and i (same (pj, pk)) splits, in this order on every rank
int grid_init(Grid* g, cflx_comm* c, int Px, int Py, int Pz);
void grid_free(Grid* g);

// ---------------------------------------------------------------- the solve engine (solve.cu)
// ---------------------------------------------------------------- iterative refinement (refine.cu)
// Device buffers of cflx_lu_refine / cflx_chol_refine, grown and never shrunk, freed with the solve cache.  gl_cols /
// gl_rows: the row of X that each local column / row of the layer-0 share multiplies (made on first use; the layout does
// not change with the matrix).
struct RefineCache {
    DevBuf<int> gl_rows, gl_cols, active;
    DevBuf<double> X, B, R, D, rhs, ratio, W;  // M x ldn each, grown together
    DevBuf<double> Xc, Xr, part, all, berr;
    // cflx_*_refine_x only: the tail of X (M x ldn) and its gathered copies, the per-column statistics of a round
    DevBuf<double> T, Xct, Xrt, stats;
};

// ---------------------------------------------------------------- equilibration and the expert drivers (equil.cu)
// The scaling an input carries (cflx_*_equilibrate), and the one the factors of that input carry on to cflx_*_svx:
// equed 'N' (none), 'R', 'C', 'B' (LU) or 'Y' (Cholesky); r / c: the row and column scales on the device (M each, every
// rank; the Cholesky's s is r), with rowcnd / colcnd (the Cholesky's scond is rowcnd).  Each record owns its scales:
// nothing but equil_record_set writes them.
struct EquilRecord {
    char equed = 'N';
    double rowcnd = 1.0, colcnd = 1.0;
    DevBuf<double> r, c;  // grown together
};
// The records of the input and of the factors, the results of the last equilibrate call (which change no record unless
// that call scaled the input), and the device work buffers of svx.  Buffers are grown, never shrunk.
struct EquilState {
    EquilRecord in, fac;
    DevBuf<double> qr, qc;  // the last call's scales (dgeequ's r, c; dpoequ's s in qr), grown together
    DevBuf<double> B, X;    // svx: M x ldn each, grown together
    DevBuf<double> growth;  // the pivot growth's maxima by column: amax (M), then fmax (M)
    DevBuf<int> ival;       // 1 int: the first zero pivot
    DevBuf<double> det;     // M + 4 doubles: the gathered diagonal, then det_grid's DetResult
};
// *dst = {equed, rowcnd, colcnd} with device copies of r and c (n each; c may be null: then only r is kept)
int equil_record_set(EquilRecord* dst, char equed, double rowcnd, double colcnd, const double* r, const double* c, int n,
                     cudaStream_t s);
// in -> fac; then, when `next_is_plain`, in becomes 'N' (a streamed next input)
int equil_pass_on(EquilState* e, int M, bool next_is_plain, cudaStream_t s);

// ---------------------------------------------------------------- random butterfly transforms (rbt.cu)
// The transform an input carries (cflx_lu_rbt: A0 <- U^T A0 V), and the one the factors of that input carry on to
// cflx_lu_rbt_solve / cflx_lu_rbt_apply_local, kept like EquilState's records: depth 0 (none) or 1 .. 4, the seed, and
// s: the device multipliers s = fl(r fl(1/sqrt 2)), U's d x M then V's d x M (every rank).
struct RbtRecord {
    int depth = 0;
    uint64_t seed = 0;
    DevBuf<double> s;
};
struct RbtState {
    RbtRecord in, fac;
};
// *dst = {depth, seed} with a copy of s (2 depth M doubles, host or device) when depth > 0
int rbt_record_set(RbtRecord* dst, int depth, uint64_t seed, const double* s, int M, cudaStream_t st);
// in -> fac; then, when `next_is_plain`, in carries no transform (a streamed next input)
int rbt_pass_on(RbtState* t, int M, bool next_is_plain, cudaStream_t s);
// r (depth x M, level l at l M) of side 0 (U) or 1 (V): r = exp((w - 0.5) / 10) with w the top 53 bits of splitmix64's
// finaliser of seed + 0x9E3779B97F4A7C15 (((2 l + side) << 32) + i + 1), in [e^-0.05, e^0.05]; pure host
void rbt_multipliers(int M, int depth, uint64_t seed, int side, double* r);
// s[i] = fl(r[i] fl(1/sqrt 2)) for i < n
void rbt_scales(const double* r, size_t n, double* s);
// The operations on a share X (ld) of L's rows: U^T, V, V^T, U on the local columns c < ncols with L.col(c) < col_lim
// (a right-hand side), or W = U^T X V on the whole Ml x ncols share (ncols = L.Nl).  Needs Ml (and for W ncols) a multiple
// of 2^depth v; su / sv: the device multipliers of U and V (depth x L.M each).  Bits as oracle/rbt_ref.py.
enum class RbtOp { UT = 0, V = 1, VT = 2, U = 3, W = 4 };
int launch_rbt(RbtOp op, double* X, int64_t ld, const Layout& L, int ncols, int col_lim, int depth, const double* su,
               const double* sv, cudaStream_t s);

// What a solve keeps between calls: prepared by the first solve after a factorisation, dropped (ready = false) by
// set_local / factor, freed with the object.  The work buffers have ldn columns and are grown, never shrunk.
struct SolveCache {
    bool ready = false;
    DevBuf<double> inv;  // per owned diagonal tile: the forward inverse blocks (v x nb, row-major nb x nb each), then
                         // the backward ones
    DevBuf<int> rows;    // row of B of each seeded local row (ranks (pi, 0, 0))
    // the transposed LU solve and the LU condition estimate, prepared on first use after solve data is prepared
    bool trans_ready = false;
    DevBuf<int> rows_id;  // identity row map by local tile row (ranks (pi, 0, 0)): P*A solved without P
    DevBuf<int> cols;     // row of B of each seeded local column (ranks (0, pj, 0))
    DevBuf<int> unperm;   // row of the solved system that lands in each row of X: X[perm[q]] = W[q] (every rank)
    DevBuf<double> B, W, Z, R, Y, X, Xg;  // grown together
    int ldn = 0;
    bool col_partials = false, col_seed = false;  // what the buffers were grown for (kept across growth)
    RefineCache rf;
};

// The triangle a diagonal-tile solve applies, and how (solve.cu diag_solve):
//   Lower:      L_tt       (forward inverses, NN)          Upper:  U_tt   (backward inverses, NN)
//   LowerT:     L_tt^T     (backward inverses, NN: the Cholesky's inv(L_jj)^T)
//   UnitLowerT: L_tt^T     (forward inverses read transposed, TN: the LU's unit L)
//   UpperT:     U_tt^T     (backward inverses read transposed, TN)
enum class Tri { Lower, Upper, LowerT, UnitLowerT, UpperT };

// Where a right-hand side enters the sweeps: B is held on the layer-0 ranks of grid column 0 (by_col = false, dst = W by
// local tile row) or of grid row 0 (by_col, dst = Z by local tile column), and dst[r] = B[rows[r]] for r < n there.
struct SolveSeed {
    bool by_col;
    const int* rows;
    int n;
    double* dst;
};

// One factor in the conflux block-cyclic layout of its grid g, as the engine reads it: tile (I, J) on rank
// (I % Px, J % Py, 0) at local tile (I / Px, J / Py) of F (layer 0, row-major, leading dimension Nl; B and X have M rows).
// A rank's NCCL rank in the grid-row communicator is pj * stride (+ pk), in the grid-column communicator pi * stride
// (+ pk).
struct SolveFactor {
    const Grid& g;
    const double* F;
    int rows;  // local rows of the tiles the sweeps read and seed
    const SubComm *row_comm, *col_comm;
    int stride;
    const double* sgn = nullptr;  // a signed Cholesky factor's S (M, device, every rank): A = F S F^T; null: S = I
};

// How a kind of handle words its state errors, after "<function>: " (callers match these texts)
struct HandleTexts {
    const char* unfactored;  // no factorisation to work on
    const char* no_input;    // before the first upload
    const char* scaled;      // format, %c: the input's equed
};

// What the LU and Cholesky handles share: the input and its working copy, the state rules between set_local,
// equilibrate and factor, the trailing-update choice, the look-ahead stream, the solve cache and the scaling records.
struct Handle : Grid {
    const HandleTexts* texts = nullptr;
    DevBuf<double> A0, A11;  // the input share and the working copy the factorisation overwrites, Ml x Nl
    bool have_input = false, factored = false;
    bool a0_is_next = false;  // A0 already holds (or is receiving) the next input (LU input streaming)
    int64_t launches = 0;
    Stream side;            // high-priority look-ahead stream (null: no overlap)
    TrailingUpdate update;  // handle_update_setup; TF32 for the factorisations of a mixed-precision driver
    bool low_prec = false;  // the factors of the last factorisation came from a TF32 update
    SolveCache sv;
    EquilState eq;  // cflx_*_equilibrate / cflx_*_svx
    RbtState rbt;   // cflx_*_rbt: the transform of the input and of the factors
    DevBuf<unsigned long long> agree;  // the words the ranks compare before a fixed factorisation or a transform
};
// grid_init, then A0 and A11 (not zeroed)
int handle_init(Handle* h, const HandleTexts* texts, cflx_comm* c, int Px, int Py, int Pz);
// the trailing update: the FP64 DMMA kernel, or the int8 digit planes with CFLX_GEMM=ozaki where a layer's contraction
// length allows.  Called after the handle's own buffers are allocated: loading the update kernels first moves those
// buffers in device memory, and the one-GPU LU step time moves with them.
int handle_update_setup(Handle* h);
// h->side, at the device's highest stream priority
int handle_side_stream(Handle* h);
// host_local into A0, waited for: a new unscaled input, without factors or a solve cache
int handle_set_local(Handle* h, const double* host_local);
// What an entry point needs of its handle's state (enter)
enum Need : unsigned {
    NEED_INPUT = 1,      // an input (set_local)
    NEED_UNSCALED = 2,   // an input that carries no scaling
    NEED_FACTORS = 4,    // a successful factorisation
    NEED_OWN_INPUT = 8,  // A0 still holds the input of that factorisation (not a queued next one)
    NEED_FP64 = 16,      // factors of an FP64 trailing update (not those a mixed-precision driver left)
};
// The prologue of every entry point `who` on a handle, after its argument checks: CFLX_ERR_STATE with "<who>: <reason>"
// unless h's state has what `need` asks for, then h's device made current
int enter(Handle* h, const char* who, unsigned need);
// the input changes, so the factors and the solve cache are dropped, as by set_local
void handle_equil_begin(Handle* h);
// the input's record changes only when the call scaled it (apply, info == 0): equed with eq.qr and c (may be null); a
// query leaves the record and its scales
int handle_equil_end(Handle* h, bool apply, int info, char equed, double rowcnd, double colcnd, const double* c);
int handle_launch_count(Handle* h, int64_t* count_out, int reset);
// COLLECTIVE (world): *same = every rank has ok and the same words, from one ncclMin over {w.., ~w.., ok}
int world_agree(Handle* h, bool ok, std::initializer_list<unsigned long long> words, bool* same);
}  // namespace cflx

// sv (cflx_lu_solve): Linv blocks forward, Uinv blocks backward; rows: row of B of each row of P*B
struct cflx_lu : cflx::Handle {
    int N = 0, Mt = 0;
    cflx::SubComm jk_comm, ik_comm;
    // device memory
    cflx::DevBuf<double> PT, PT2, W, LT, A01raw, U, tmp, A00, A00T, Uinv, LinvT, candH, S, W2, bcast, Cbuf, xbuf;
    cflx::DevBuf<int> gri, gri_tmp, igri, perm, gpivots, tagsH, tagsS, hist, plan_mem, idx_buf;
    cflx::MovePlan plan{};
    cflx::PanelWorkspace pws{};
    int64_t ldp_max = 0;
    cflx::PinnedBuf<int> h_npiv;
    bool time_gemm = false;
    // double-buffered input streaming (cflx_lu_queue_next_local): the upload of the NEXT matrix overlaps this factorisation
    const double* next_host = nullptr;
    cflx::Stream copy;
    cflx::Event ev_a0_read, ev_upload;
    double gemm_ms = 0, gemm_flops = 0;
    double phase_ms[cflx::PH_COUNT] = {0};
    // non-serialising timeline (profiling mode 2): event pairs recorded on the launching stream, resolved after the run
    struct TlRec { int region, side, ev; };
    std::vector<cflx::Event> tl_pool;
    std::vector<TlRec> tl_recs;
    struct TlSpan { int region, side; float start_ms, ms; };  // resolved: start relative to the first recorded event
    std::vector<TlSpan> tl_spans;                             // one per region instance, in launch order
    double region_ms[2][cflx::RG_COUNT] = {{0}};   // [main / side stream][region]
    int region_cnt[2][cflx::RG_COUNT] = {{0}};
    int prof_mode = 0;                              // 0 off, 1 serialising phase timers, 2 timeline
    std::vector<cflx::Event> ev;
    std::vector<char> ev_used;
    cflx::Event ev_fork, ev_join, ev_npiv;
    // hist holds the permutation of a completed factorisation (cleared when one starts, set when it completes)
    bool perm_done = false;
    // cflx_lu_factor_fixed: the plan's fixed-order flag, the prescribed order (host and device, M each), this rank's
    // pivot count per step, the tiny-pivot threshold, and the device record {replacements, first zero pivot, its min
    // operand} (4 ints) and the tile kernel's scratch (getrf_nopiv_scratch(v)); the device buffers are made by the first
    // fixed call
    bool fixed = false;
    std::vector<int> fix_perm_h, fix_npiv;
    double fix_tiny = 0.0;
    cflx::DevBuf<int> fix_perm, fix_rec;
    cflx::DevBuf<double> fix_ws;
    ~cflx_lu();  // the handle's device made current, the sub-communicators destroyed, then the members freed
};

namespace cflx {
// validate.cu
int redistribute_pivoted_rows(cflx_lu* lu, const std::vector<int>& hist, bool factors, const double* src, double* dst);
int lu_residual_grid(cflx_lu* lu, const std::vector<int>& hist, double* abs_out, double* rel_out);
// Step t of lu_residual_grid's sweep on one layer-0 share C of the packed factors (L's layout, leading dimension Nl), each
// a no-op on the ranks that do not hold the block:
//   extract_l (grid column t % Py): LT[c][r] = L(global row of r, t v + c) for the local rows r from the first local tile
//             row with a global index >= t: the multiplier below the diagonal, 1 on it, 0 above;
//   extract_u (grid row t % Px): U[r][lc] = U(t v + r, global column of lc) for the local columns lc from the first
//             local tile column with a global index >= t: the entry on and above the diagonal, 0 below.
int launch_lu_extract_l(const double* C, const Layout& L, int t, double* LT, int64_t ldp, cudaStream_t s);
int launch_lu_extract_u(const double* C, const Layout& L, int t, double* U, int64_t ldu, cudaStream_t s);

// The Cholesky panel buffers' leading dimension (LT, PT, W, and the slot of each broadcast piece: a piece stride of
// v chol_panel_ld), and the leading dimension of piece p of the panel of global tiles >= gfirst: its active rows, even,
// >= 2 (what is broadcast is v chol_piece_ld doubles)
inline int64_t chol_panel_ld(int Ml) { return round_up(Ml, 2) + 2; }
inline int chol_piece_ld(const Layout& L, int gfirst, int p) {
    const int rows = L.Ml - first_local_tile(gfirst, p, L.Px) * L.v;
    return (int)std::max<int64_t>(2, round_up(std::max(rows, 0), 2));
}
// chol.cu, the kernels of the timed column operand and of cflx_chol_validate.
//   gather_cols: Bc[c][t v + x] = piece p = j % Px of G (piece p at G + p piece_stride, [v][ld_p] with ld_p its active
//                rows from global tile gfirst on, rounded up to even, >= 2) at row (j / Px - first_p) v + x, for the
//                ntiles local column tiles t from lj0 (global tile j = (lj0 + t) Py + pj)
//   sumsq_lower: *out += the sum of squares of X's entries in the lower triangle of the real tiles (global row >= global
//                column, global row < Nt v); partials: SUMSQ_PARTIALS doubles of scratch
//   extract_l_panel_T: PT[c][r] = A[row0 + r][col0 + c] for r < n, c < v where the global row of local row row0 + r is
//                >= the global column t v + c, else 0
//                sg (may be null): Bc's row c times sg[c] (the signs of the step, cflx_chol_factor_ldlt)
int launch_gather_cols(const double* G, int64_t piece_stride, double* Bc, int64_t ldb, int v, int Px, int Py, int pj,
                       int lj0, int ntiles, int gfirst, int Ml, cudaStream_t s, const double* sg = nullptr);
int launch_sumsq_lower(const double* X, const Layout& L, double* partials, double* out, cudaStream_t s);
int launch_extract_l_panel_T(const double* A, int64_t lda, int row0, int col0, int n, const Layout& L, int t, double* PT,
                             int64_t ldp, cudaStream_t s);

// solve.cu: the solve engine.  Every function returns CFLX_OK or an error code; all work goes on f.comm->stream.
// grow the work buffers to ldn columns: B (M rows) on rank (pi, 0, 0), W (Ml) and R, Y (v) where `work`, Z (Nl) where
// `work && col_partials`, X (M) on every rank.  col_seed: also B on rank (0, pj, 0) and Xg (M) on every rank.  What was
// once asked for stays allocated.
int solve_cache_grow(SolveCache* sc, const SolveFactor& f, int ldn, bool work, bool col_partials, bool col_seed = false);
// the inverses of the nb x nb diagonal blocks of every owned diagonal tile, into sc->inv (freed and allocated again here).
// lower: the tile is L with its own diagonal and zeros above, inverted as A00 = L^T; otherwise it is L\U with a unit L.
int solve_inverses(SolveCache* sc, const SolveFactor& f, bool lower);
// solve_inverses' work on one diagonal tile T (v x v at leading dimension ld): the inverse blocks into inv (2 v nb: the
// forward half, then the backward one), with scratch tile (v x v) and linvT (v x nb)
int solve_tile_inverses(const double* T, int64_t ld, int v, int nb, bool lower, double* inv, double* tile, double* linvT,
                        cudaStream_t s);
// Y (v x ldn) = T^-1 R by the nb-block sweep over one diagonal tile ftt (leading dimension Nl) with its inverse blocks
// tile_inv (solve_tile_inverses' inv); tri says which triangle of ftt is T and how it is read.  R is overwritten.
int diag_solve(const double* tile_inv, const double* ftt, int64_t Nl, int v, int nb, Tri tri, double* R, double* Y,
               int ldn, cudaStream_t s);
// *dst = rows (allocated on first use), waited for
int solve_set_rows(DevBuf<int>* dst, const std::vector<int>& rows, cudaStream_t s);
// zero X, W and Z, and on the ranks holding B (`at`): at.dst[r] = B[at.rows[r]] for r < at.n; B is a host or device array
int solve_seed(SolveCache* sc, const SolveFactor& f, int ldn, int nrhs, const double* B, int ldb, const SolveSeed& at);
// row-partial sweep over the tile diagonal: forward with the lower triangle (NN), backward with the upper one (NN).  The
// diagonal owner keeps each solved tile t at tile t / keep_div of `keep`; with clear_row, keep is W and the other layer-0
// ranks of the grid row zero their copy of that tile.  [t_lo, t_hi) (t_hi < 0: Nt): the diagonal tiles the sweep visits,
// in its direction; the default is every tile.
int solve_row_sweep(SolveCache* sc, const SolveFactor& f, int ldn, bool forward, double* keep, int keep_div,
                    bool clear_row, int t_lo = 0, int t_hi = -1);
// column-partial sweep over the tile diagonal (Z by local tile column, the factor read transposed): backward with L^T
// (tri LowerT or UnitLowerT; update of the local columns t_lo <= gj < t), forward with U^T (UpperT; update of the
// columns gj > t).  The diagonal owner keeps each solved tile t at tile t / keep_div of `keep`; with clear_col, keep is Z
// and the other layer-0 ranks of the grid column zero their copy of that tile.  Ranks pk != 0 join the collectives only.
// [t_lo, t_hi) as solve_row_sweep.
int solve_col_sweep(SolveCache* sc, const SolveFactor& f, int ldn, bool forward, Tri tri, double* keep, int keep_div,
                    bool clear_col, int t_lo = 0, int t_hi = -1);
// between the two sweeps of a signed factor (f.sgn): Y <- S Y on the Y_t the row sweep kept in Z (by local tile column;
// every other entry of Z is zero then), on layer 0; nothing without f.sgn
int solve_apply_signs(SolveCache* sc, const SolveFactor& f, int ldn);
// its kernel on one share: Z[r][j] *= sgn[L.col(r)] for r < L.Nl with L.col(r) < L.M, j < ldn (Z: Nl x ldn, device)
int launch_solve_signs(double* Z, int ldn, const Layout& L, const double* sgn, cudaStream_t s);
// X (nrhs columns, ldx; host or device) = the world sum of the owners' tiles of sc->X, copied when X is not null;
// synchronises.
// unperm (M rows, every rank): row i of X is row unperm[i] of that sum.
int solve_finish(SolveCache* sc, const SolveFactor& f, int ldn, int nrhs, double* X, int ldx, const int* unperm = nullptr);
// Hager-Higham estimate of ||inv(A)||_1 for an order-n A, as LAPACK's dlacn2 runs it (x = 1/n, at most 5 iterations,
// the sign-vector test, the final alternating vector).  apply(kase, x) overwrites the host vector x with inv(A) x
// (kase 1) or inv(A)^T x (kase 2) and returns a status.  Pure host logic on x: ranks that pass bit-identical vectors
// make the same choices, so every rank calls `apply` the same number of times with the same kase.
int estimate_inv_norm1(int n, const std::function<int(int, double*)>& apply, double* est);
// the collective 1-norm of the matrix whose layer-0 shares are A (g's layout), into *anorm (every rank).
// lower_sym: only the lower triangle of the real tiles (global tile index < Nt) is stored and the matrix is its symmetric
// completion; otherwise every local entry of the M x M matrix counts.  Deterministic: no floating-point atomics.
int norm1_grid(const Grid& g, const double* A, bool lower_sym, double* anorm);
// norm1_grid's and norminf_grid's per-share passes on one layer-0 share A (L's layout, M-vectors by global index):
//   norm1_share: out[g] = this share's part of global column g's sum of |a| (lower_sym as norm1_grid), for every g < M,
//                from the per-CTA partials colp (ncp x Nl) and, when lower_sym, rowp (nrp x Ml) (norm1_partials)
//   norminf_share: out[g] = the sum of |a| over this share's row g, for the global rows it holds; out is not written
//                elsewhere
void norm1_partials(const Layout& L, int* ncp, int* nrp);
int launch_norm1_share(const double* A, const Layout& L, bool lower_sym, double* colp, double* rowp, double* out,
                       cudaStream_t s);
int launch_norminf_share(const double* A, const Layout& L, double* out, cudaStream_t s);
// rcond = (1 / ainvnm) / anorm as LAPACK's dgecon / dpocon form it; 0 when anorm is 0 or the estimate is not finite
double rcond_from(double anorm, double ainvnm);

// LAPACK's dlacn2 as a reverse-communication step (Higham, ACM TOMS 14 (1988) 381-396, Algorithm 4.1 with dlacn2's
// safeguards): start(n) sets x = 1/n and kase = 1; the caller overwrites x with A x (kase 1) or A^T x (kase 2) and calls
// step(), which sets the next x and kase, until kase == 0 and est is the estimate of ||A||_1.  The sign vector is +1 for
// x >= 0, idamax takes the first index of the largest |x|, and the sums of |x| run in index order.  Pure host logic:
// callers that pass bit-identical vectors take the same steps.
struct Lacn2 {
    int n = 0, kase = 0, jump = 0, j = 0, iter = 0;
    double est = 0.0;
    bool pending = false;  // a product was written into x and step() has not taken it yet (refine_run's bookkeeping)
    std::vector<double> x, v;
    std::vector<int> isgn;
    void start(int n);
    int step();
};

// What refine_run needs of a factorisation: its grid, the input's layer-0 share, and the solves.
// solve(transposed, nrhs, B, ldb, X, ldx) overwrites X with inv(op A) B (transposed: inv(op A)^T B); B and X are host or
// device arrays of M rows; it synchronises the stream.  symmetric: both kinds are the same solve.
struct RefineOp {
    const Grid& grid;
    const double* A;
    ResidMode mode;
    bool symmetric;
    std::function<int(bool, int, const double*, int, double*, int)> solve;
};
// LAPACK dgerfs / dporfs on the grid (collective): X (host or device, M x nrhs, ldx) refined in place from B (host or
// device), ferr (may be null: no estimator) and berr (may be null) per column.  Every column runs LAPACK's own decisions, all in lockstep.
int refine_run(RefineCache* rc, const RefineOp& op, int nrhs, const double* B, int ldb, double* X, int ldx, double* ferr,
               double* berr);
// LAPACK dsgesv / dsposv's refinement loop on the grid (collective), after a factorisation with a TF32 update: X =
// op.solve(B), then R = B - op(A) X in FP64 from op.A and, until every column has ||r||_inf <= ||x||_inf anorm eps
// sqrt(M) (eps = 2^-53), X += op.solve(R), at most itmax times.  *iter = the corrections taken when the loop converged,
// MIXED_NO_CONVERGENCE when it did not within itmax or a norm is not finite.  berr (may be null): ||r||_inf / (anorm
// ||x||_inf) per column of the last residual.  X (host or device, ldx) is written in every case.
constexpr int MIXED_ITMAX = 30;               // dsgesv's ITERMAX
constexpr int MIXED_NO_CONVERGENCE = -31;     // dsgesv's -ITERMAX - 1
constexpr int MIXED_LOW_PREC_FAILED = -3;     // the low-precision factorisation met a zero or non-positive pivot
int mixed_run(RefineCache* rc, const RefineOp& op, double anorm, int itmax, int nrhs, const double* B, int ldb, double* X,
              int ldx, int* iter, double* berr);
// the same backward errors of a given X (host or device)
int mixed_berr(RefineCache* rc, const RefineOp& op, double anorm, int nrhs, const double* B, int ldb, const double* X,
               int ldx, double* berr);
// One column of LAPACK's dla_gerfsx_extended / dla_porfsx_extended: its precision state and the normwise (x) and
// componentwise (z) convergence states, with LAPACK's initial values.  round() takes the statistics of one round,
// {normy, normx, normdx, dz_z, ymin} (refine.cu column_stats_kernel), and returns what to do with the correction dy:
// 0 stop (no update), 1 y += dy, 2 (y, y_tail) += dy in double-double.  finish() sets the error estimates.
struct RefineXColumn {
    enum { UNSTABLE = 0, WORKING = 1, CONV = 2, NOPROG = 3 };
    enum { EXTRA_RESIDUAL = 1, EXTRA_Y = 2 };
    int x_state = WORKING, z_state = UNSTABLE, y_prec = EXTRA_RESIDUAL;
    bool done = false;
    double dx_x = INFINITY, dz_z = INFINITY, prev_normdx = INFINITY, prev_dz_z = INFINITY;
    double dxratmax = 0.0, dzratmax = 0.0, final_dx_x = INFINITY, final_dz_z = INFINITY;
    double err_norm = 0.0, err_comp = 0.0;
    int round(const double st[5], double rcond, bool ignore_cwise, int cnt, int M);
    void finish();
};
// LAPACK dgerfsx / dporfsx on the grid (collective), after the caller's zero-pivot check: X (host or device, M x nrhs,
// ldx) refined in place from B with residuals in double-double (launch_residual_x); d (device, M; null: ones) the scales
// of the unscaled solution diag(d) y; rcond the dgecon / dpocon estimate the precision switch uses.  Per column: berr
// (may be null), err_norm and (when cwise) err_comp as nrhs x 3 {trust, err, rcond}.  *info = M + j for the first
// column j (1-based) with a bound set to 1 for an ill-conditioned problem, else 0.
int refine_x_run(RefineCache* rc, const RefineOp& op, int nrhs, const double* B, int ldb, double* X, int ldx,
                 const double* d, double rcond, bool cwise, double* berr, double* err_norm, double* err_comp, int* info);
// The residual kernels (refine.cu).  From layer 0's share A (L's layout, lda = Nl even, 16-byte aligned, v % 4 == 0)
// and X gathered by local column (Xc, Nl x nrhs) or by local row (Xr, Ml x nrhs), both with leading dimension ldx:
//   NN:       P = A Xc, Q = |A| |Xc| by local row (Ml rows);
//   TN:       P = A^T Xr, Q = |A|^T |Xr| by local column (Nl rows);
//   SymLower: the stored lower triangle of the real tiles (global tile index < Nt): the NN product of the entries
//             with global row >= global column into rows [0, Ml), the TN product of those with global row > global
//             column into rows [Ml, Ml + Nl).  Nothing else is read.
// P and Q have leading dimension ldo.  Deterministic: no floating-point atomics.
int launch_residual(ResidMode mode, const double* A, const Layout& L, const double* Xc, const double* Xr, int64_t ldx,
                    int nrhs, double* P, double* Q, int64_t ldo, cudaStream_t s);
// Their double-double counterparts (SIMT FP64, Dot2): Hi + Lo = op(A) (X + Xt) in the same modes, layouts and masks, from
// the head Xc / Xr and the tail Xct / Xrt (either tail may be null: zero).  The entries are combined in a fixed order
// (lanes, then warps, by double-double additions): deterministic, no atomics.
int launch_residual_x(ResidMode mode, const double* A, const Layout& L, const double* Xc, const double* Xct,
                      const double* Xr, const double* Xrt, int64_t ldx, int nrhs, double* Hi, double* Lo, int64_t ldo,
                      cudaStream_t s);
// The refinement's assembly of the grid's partials (refine.cu).  For global row g (tile T) every rank adds, in this order,
// the NN partials of the ranks (T % Px, pj, 0), pj ascending, then the TN partials of the ranks (pi, T % Py, 0), pi
// ascending, each out of its chunk of `all`.
struct AssembleArgs {
    const double* all;  // the partials of every world rank, `chunk` doubles apart: rows of 2 ldn (P, then Q)
    int64_t chunk;
    int Ml, Nl, ldn, nrhs, M;
    bool nn, tn;           // which partials a rank holds: NN rows [0, Ml), then TN rows [nn ? Ml : 0, + Nl)
    int v, Px, Py, Pz;
    const double* B;       // [M x ldn]
    double *R, *ratio, *W;  // [M x ldn]: b - op(A) x, the backward-error ratio, dgerfs' w
    double safe1, safe2, nzeps;
    bool lin_berr;      // refine_x: ratio = (|r_i| + safe1) / s_i where s_i != 0, else 0 (LAPACK dla_lin_berr); no W
    double* Q;          // refine_x (may be null): |op(A)| |x|
};
// dgerfs' safe1 = (M + 1) safmin, safe2 = safe1 / eps and (M + 1) eps of an order-M system
void refine_safe(int M, double* safe1, double* safe2, double* nzeps);
// assemble (extended: the double-double partials, R = b - their sum rounded once; otherwise R, ratio and W or Q)
int launch_assemble(const AssembleArgs& a, bool extended, cudaStream_t s);
// The per-column steps on M x ldn arrays, nrhs columns:
//   column_max:   berr[c] = max over the rows of ratio[:, c] (NaN wins)
//   column_stats: out[c][0..4] = {max |y|, max |y| d, max |dy| d, max |dy| / |y| (+inf where y = 0 != dy, 0 where
//                 y = dy = 0), min |y|} (d null: ones; NaN wins)
//   select_cols:  out[:, c] = active[c] ? in[:, c] : 0;  add_cols: X[:, c] += D[:, c] where active[c]
//   update_x:     how[c] 1: Y += DY; 2: (Y, T) += DY as LAPACK's dla_wwaddw; 0: nothing
constexpr int REFINE_NSTAT = 5;
int launch_column_max(const double* ratio, int M, int ldn, int nrhs, double* berr, cudaStream_t s);
int launch_column_stats(const double* Y, const double* DY, const double* d, int M, int ldn, int nrhs, double* out,
                        cudaStream_t s);
int launch_select_cols(const double* in, const int* active, int M, int ldn, double* out, cudaStream_t s);
int launch_add_cols(double* X, const double* D, const int* active, int M, int ldn, cudaStream_t s);
int launch_update_x(double* Y, double* T, const double* DY, const int* how, int M, int ldn, cudaStream_t s);
// The expert drivers' solve (equil.cu), COLLECTIVE: B (host or device, M x nrhs) to the device, pre on its rows, X =
// op.solve(false, B), refine(B, ldb, X, ldx) on the device X in place, post on the rows of X, X out; synchronises.  A
// row transform (empty: none) runs in place on an M x n device array with leading dimension ld, on the grid's stream.
using RowTransform = std::function<int(double* X, int64_t ld, int n)>;
using SvxRefine = std::function<int(const double*, int, double*, int)>;
int svx_tail(EquilState* e, const RefineOp& op, int nrhs, const double* B, int ldb, double* X, int ldx,
             const RowTransform& pre, const RowTransform& post, const SvxRefine& refine);
// rbt.cu.  The transform h's factors carry, as a row transform of an M-row device array (the replicated right-hand sides)
RowTransform rbt_rows(const Handle& h, RbtOp op);
// Not collective.  One of the factors' butterflies on the rows of this rank's right-hand side share B_local (host or
// device, ldb >= rhs_local_cols: checked by the caller), in the name of `who`; CFLX_ERR_STATE when the factors carry no
// transform (`rbt_call` names the call that makes one)
int rbt_apply_local(const char* who, const char* rbt_call, Handle* h, RbtOp op, int nrhs, double* B_local, int ldb);
// COLLECTIVE within each layer.  The symmetric completion of the stored lower triangle of the real tiles of the shares
// A (h's layout): tile (I, J), I < J < Nt, receives tile (J, I)^T from rank (J % Px, I % Py) -- transposed in place
// when that is this rank, else packed per peer and exchanged in one group of ncclSend / ncclRecv (staging buffers of
// the exchanged tiles only) -- and every diagonal tile's upper triangle its lower one transposed.  Nothing else is
// written.  Synchronises.
int sym_mirror(const Grid& h, double* A);
// The solve and refinement of cflx_lu_svx / cflx_chol_svx (equil.cu), COLLECTIVE: B (host or device) to the device, its
// rows scaled by pre (may be null), X = op.solve(false, B), refine_run, the rows of X scaled by post (may be null), X out;
// when post is not null, ferr is divided by cnd.  Then *info = M + 1 when rcond < 2^-53 (dgesvx / dposvx: the matrix is
// singular to working precision), else 0.
int svx_run(EquilState* e, RefineCache* rc, const RefineOp& op, int nrhs, const double* B, int ldb, double* X, int ldx,
            double* ferr, double* berr, const double* pre, const double* post, double cnd, double rcond, int* info);
// The same steps for cflx_lu_svxx / cflx_chol_svxx, with refine_x_run (d, rcond, cwise, berr, err_norm, err_comp and
// info as there) in place of refine_run.  The bounds already refer to the unscaled x: nothing is divided.
int svxx_run(EquilState* e, RefineCache* rc, const RefineOp& op, int nrhs, const double* B, int ldb, double* X, int ldx,
             const double* pre, const double* post, const double* d, double rcond, bool cwise, double* berr,
             double* err_norm, double* err_comp, int* info);

// norm.cu: the collective infinity-norm (maximum row sum) of the M x M matrix whose layer-0 shares are A (every local
// entry counts), into *anorm (every rank).  Deterministic: no floating-point atomics.
int norminf_grid(const Grid& g, const double* A, double* anorm);

// equil.cu.  Per-share kernels (layer 0's share A in L's layout); each writes an M-vector indexed by global row / column
// with zeros where this share holds nothing:
//   rowmax[g] = max |a_gj| over this share's row g;  colmax[g] = max |a_ig| r_i over this share's column g;
//   diag[g] = a_gg where this share holds the diagonal entry (real tiles, global tile index < Nt).
// The apply passes scale A in place: equed 'R' a_ij = r_i a_ij, 'C' c_j a_ij, 'B' (c_j r_i) a_ij, over every local entry;
// sym_apply: (s_j s_i) a_ij over the stored lower triangle of the real tiles only.
int equil_row_max(const double* A, const Layout& L, double* rowmax, cudaStream_t s);
int equil_col_max(const double* A, const Layout& L, const double* r, double* colmax, cudaStream_t s);
int equil_diag(const double* A, const Layout& L, double* diag, cudaStream_t s);
// COLLECTIVE: d (M doubles, device) = the diagonal of the layer-0 shares A on every rank, bit-identical (equil_diag on
// layer 0, zeros on the other layers, one ncclSum over the world: one non-zero contributor per element)
int diag_grid(const Grid& g, const double* A, double* d);
int equil_apply(double* A, const Layout& L, const double* r, const double* c, char equed, cudaStream_t s);
int equil_sym_apply(double* A, const Layout& L, const double* sc, cudaStream_t s);
// On a share F of L\U (and A of the input): *zero_pivot = min(1 + g) over the global diagonal entries g < M the share
// holds with F_gg == 0 (INT_MAX: none).
int equil_zero_pivot(const double* F, const Layout& L, int* zero_pivot, cudaStream_t s);
// The pivot growth's maxima by global column g < ncols, out = {amax (M), fmax (M)} with zeros where the share holds
// nothing.  LU (!sym, F = L\U): amax_g = max |a_ig| over every row, fmax_g = max |f_ig| over the rows i <= g.  Cholesky
// (sym, F = L, both the stored lower triangles): the real tiles' entries with g <= i < ncols of A and of F.  Nothing
// outside these masks is read.
int equil_growth_cols(const double* F, const double* A, const Layout& L, bool sym, int ncols, double* out,
                      cudaStream_t s);
// the first exactly zero U(k,k) of the layer-0 shares F of L\U on the grid, COLLECTIVE (ncclMin over the world): *info =
// k (1-based), or 0 when there is none; the same on every rank
int zero_pivot_grid(const Grid& g, EquilState* e, const double* F, int* info);
// LAPACK dgeequ, or dgeequb when pow2 (+ dlaqge when `apply`) on the grid, COLLECTIVE: the scales into e->qr / e->qc (no
// record changes) and the host results; r_out / c_out (M, may be null).  Scales are applied only when info == 0.
int geequ_grid(const Grid& g, EquilState* e, double* A, bool apply, bool pow2, double* r_out, double* c_out,
               double* rowcnd, double* colcnd, double* amax, char* equed, int* info);
// LAPACK dpoequ, or dpoequb when pow2 (+ dlaqsy, UPLO = 'L', when `apply`) on the grid, COLLECTIVE: s into e->qr (no
// record changes)
int poequ_grid(const Grid& g, EquilState* e, double* A, bool apply, bool pow2, double* s_out, double* scond,
               double* amax, char* equed, int* info);
// COLLECTIVE: equil_growth_cols on layer 0 (zeros on the other layers), one ncclMax over the world, and the host copy h
// = {amax (M), fmax (M)}, bit-identical on every rank
int growth_cols_grid(const Grid& g, EquilState* e, bool sym, const double* F, const double* A, int ncols,
                     std::vector<double>& h);
// dla_gerpvgrw / dla_porpvgrw from growth_cols_grid's h: the minimum of 1 and of amax_j / fmax_j over j < ncols with
// fmax_j != 0
double rpvgrw_cols(const std::vector<double>& h, int M, int ncols);
// The reciprocal pivot growth of the LU on the grid, COLLECTIVE: F is L\U and A the input (both layer-0 shares of the
// M x M matrix).  info = 1 + the first global k with U(k,k) == 0 (0: none); over the global columns < (info ? info : M),
// rpvgrw is dgesvx's max |A| / max |triu(U)| (1 when the denominator is 0), or with per_column dgesvxx's dla_gerpvgrw.
int pivot_growth_grid(const Grid& g, EquilState* e, const double* F, const double* A, bool per_column, double* rpvgrw,
                      int* info);
// the svx work buffers for nrhs columns (ldn = round_up(nrhs, 8)): e->B and e->X, M x ldn
int equil_grow(EquilState* e, int M, int ldn);
// X[i][j] *= d[i] for i < M, j < n (ld), on the device
int launch_scale_rows(double* X, int64_t ld, int M, int n, const double* d, cudaStream_t s);

// ---------------------------------------------------------------- the explicit inverse (inverse.cu)
// Columns of the inverse per block: a whole number of tiles near this width (all of M when M is smaller).  Measured at
// N = 16384, v = 256 among 256 .. 2048 (DESIGN §7f).
#ifndef CFLX_INV_NC
#define CFLX_INV_NC 2048
#endif
int inverse_block_cols(int M, int v);
// LU: inv(A) = inv(P A) P from L\U, column q of inv(P A) landing in column perm[q] (every entry of every share is written).
// Cholesky: dpotri's lower triangle from L, column c landing in column c on the tiles on and below the diagonal of the real
// tiles (global tile index < Nt); every other entry is set to zero.
enum class InvKind { LU, Chol };
// The per-share kernels (L: the layout of the share, global indices < L.M):
//   seed:    W[r][j] = (L.row(r) == c0 + j && j < nc) for r < rows, j < ldn (the identity block of columns c0 .. c0 + nc - 1)
//   scatter: column j < nc of X (M x ldx, by global row) into the share's column of block column c0 + j
//            (LU: global column perm[c0 + j], every local row; Cholesky: global column c0 + j, the real tiles on and
//            below the diagonal only)
//   zero:    (Cholesky) zero every entry of the share the scatter never writes
int launch_inverse_seed(double* W, int ldn, const Layout& L, int rows, int c0, int nc, cudaStream_t s);
int launch_inverse_scatter(InvKind kind, const double* X, int ldx, int c0, int nc, const int* perm, const Layout& L,
                           double* out, cudaStream_t s);
int launch_inverse_zero(const Layout& L, double* out, cudaStream_t s);
// COLLECTIVE.  The block loop: per block of nc = inverse_block_cols columns, seed, the sweeps (with the tile ranges
// that skip the block's zero rows), solve_finish's all-reduce and the scatter into Ainv (Ml x Nl, host or device, may be
// null).  The solve cache must be prepared; perm: the LU's permutation on the device (every rank).
int inverse_run(SolveCache* sc, const SolveFactor& f, InvKind kind, const int* perm, double* Ainv);

// ---------------------------------------------------------------- distributed right-hand sides (solve_local.cu)
// The local columns of an M x nrhs right-hand side share on a grid with Py grid columns: v * ceil(ceil(nrhs / v) / Py)
int rhs_local_cols(int nrhs, int v, int Py);
// The local rows a distributed solve reads and writes: every row (LU), or those before the first local tile with a
// global index >= Nt (Cholesky, chol)
int solve_local_rows(const Layout& L, bool chol);
// The per-share kernels (L: the layout of the share; B / X row-major with leading dimensions ldb / ldx):
//   pack:    Bk (M x ldn, by global row) zeroed, then Bk[L.row(r)][j] = B[r][local column of c0 + j] for r < rows, j < w
//            and the block columns this share holds (B null: zeros only)
//   scatter: X[r][local column of c0 + j] = Xk[L.row(r)][j] for the same entries
int launch_solve_local_pack(const double* B, int64_t ldb, const Layout& L, int rows, int c0, int w, double* Bk, int ldn,
                            cudaStream_t s);
int launch_solve_local_scatter(const double* Xk, int ldn, const Layout& L, int rows, int c0, int w, double* X, int64_t ldx,
                               cudaStream_t s);
// A distributed solve's shares after solve_local_args: B null on the layers pk != 0 (never read there); *_dev: device
// memory of this rank's device, else host memory
struct SolveLocalArgs {
    int nrhs;
    const double* B;
    int ldb;
    bool b_dev;
    double* X;
    int ldx;
    bool x_dev;
};
// *dev: p is device (or managed) memory, which must be on this rank's device (else CFLX_ERR_ARG in the name of `who`)
int share_kind(const char* who, const Grid& g, const void* p, const char* what, bool* dev);
// The right-hand sides of the replicated solves (M x nrhs, leading dimensions ldb / ldx): CFLX_ERR_ARG in the name of
// `who` unless nrhs >= 1, B is set, ldb >= nrhs, X is set (when x_required) and ldx >= nrhs (when X is set)
int rhs_args(const char* who, int nrhs, const double* B, int ldb, const double* X, int ldx, bool x_required);
// CFLX_ERR_ARG in the name of `who` for nrhs < 1, a NULL B on layer 0, ldb (layer 0) or ldx (X set) below
// rhs_local_cols, X == B with ldx != ldb, or device memory of another device; CFLX_OK with *a filled otherwise.  No
// collective.
int solve_local_args(const char* who, const Grid& g, int nrhs, const double* B, int ldb, const double* X, int ldx,
                     SolveLocalArgs* a);
// solve(w, Bk, ldn, &Xk): the sweeps on the assembled block Bk (M x ldn device, w columns, the same on every rank), the
// solution left in *Xk (M x ldn device, the same on every rank)
using BlockSolve = std::function<int(int, const double*, int, const double**)>;
// COLLECTIVE.  The block loop of cflx_lu_solve_local / cflx_chol_solve_local: per block of inverse_block_cols columns,
// pack, the world all-reduce that assembles the block, solve, and the scatter into X (may be null); synchronises.
int solve_local_run(const Grid& g, int rows, const SolveLocalArgs& a, const BlockSolve& solve);

// ---------------------------------------------------------------- the determinant (det.cu)
constexpr int DET_THREADS = 256;  // the one CTA of the product; part of its order (oracle/det_ref.py)
// The exact-range product of an M-vector: |prod| = mant 2^exp, mant in [0.5, 1) (NaN / 0 as first_zero and nonfinite
// say); neg: the parity of the negative entries; first_zero: 1 + the first zero entry of d, 0 when none; nonfinite: an
// entry that is not finite (or a zero divisor) comes before the first zero.
struct DetResult {
    double mant;
    long long exp;
    int neg, first_zero, nonfinite, pad;
};
// the product kernel on device vectors (s1, s2 may be null), into *out (device)
int launch_det(const double* d, const double* s1, const double* s2, int n, bool square, DetResult* out, cudaStream_t s);
// COLLECTIVE: the diagonal of the layer-0 shares F gathered by diag_grid, its product (squared when `square`, divided by
// the products of s1 and s2 when given: device M-vectors, every rank) and the host copy *res, the same bits on every rank
int det_grid(const Grid& g, EquilState* e, const double* F, bool square, const double* s1, const double* s2,
             DetResult* res);
// log |det| from the pair: -inf with a zero, NaN with a non-finite entry
double det_log(const DetResult& r);
}  // namespace cflx
