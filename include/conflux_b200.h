/*
 * include/conflux_b200.h -- C ABI of the H100-native CONFLUX LU hot path (libconflux_b200.so).
 *
 * This is the drop-in boundary for ONE path of eth-cscs/conflux: conflux::LU_rep<double> and the parts of
 * conflux::lu_params<double> it needs.  Plain pointers and sizes only; every function returns 0 on success or
 * a negative status code (never throws, never aborts); cflx_last_error() gives the message of the last failure
 * on the calling thread; the message of a refused call (CFLX_ERR_ARG, CFLX_ERR_STATE) starts with the name of the function
 * and names the condition that failed.  SPMD like the reference: one host thread (or process) per rank = per GPU; every
 * entry point that is marked COLLECTIVE must be called by all ranks of the grid in the same order.
 *
 * Reference interfaces replaced (file:line relative to the reference repository):
 *   MPI_Comm / MPI_Init / MPI_Cart_create ............ src/conflux/lu/lu_params.hpp:85-108   -> cflx_comm_*
 *   lu_params<T>::initialize (sizes, grid, comms) .... src/conflux/lu/lu_params.hpp:49-138   -> cflx_lu_create
 *   lu_params<T>::get_p_grid ......................... src/conflux/lu/lu_params.hpp:21-47    -> cflx_auto_grid
 *   lu_params<T>::InitMatrix (seeded generator) ...... src/conflux/lu/lu_params.hpp:364-375  -> cflx_init_matrix_host
 *   lu_params<T>::data (local tiles, ld = Nl) ........ src/conflux/lu/layout.cpp:95-109      -> cflx_lu_set_local
 *   LU_rep<T>(gv, C, permutation) main loop .......... src/conflux/lu/conflux_opt.hpp:343-1827 -> cflx_lu_factor
 *   validation outputs C / permutation ............... src/conflux/lu/conflux_opt.hpp:1660-1771,1822 -> cflx_lu_get_factors
 * There is no CPU fallback: without a CUDA device every device entry point returns CFLX_ERR_NO_DEVICE.
 */
#ifndef CONFLUX_B200_H
#define CONFLUX_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
    CFLX_OK = 0,
    CFLX_ERR_ARG = -1,         /* invalid argument */
    CFLX_ERR_CUDA = -2,        /* CUDA runtime failure */
    CFLX_ERR_NCCL = -3,        /* NCCL failure */
    CFLX_ERR_UNSUPPORTED = -4, /* shape/grid outside the supported envelope (Px != Py, v % 4, ...) */
    CFLX_ERR_STATE = -5,       /* call order violated (e.g. get_factors before factor) */
    CFLX_ERR_NO_DEVICE = -6    /* no CUDA device visible: the library refuses to run (no CPU fallback) */
} cflx_status;

typedef struct cflx_comm cflx_comm; /* process grid handle: one per rank, owns the NCCL communicators */
typedef struct cflx_lu cflx_lu;     /* one factorisation plan: sizes, device buffers, pivot history */

#define CFLX_UNIQUE_ID_BYTES 128

const char* cflx_last_error(void);
const char* cflx_version(void);
int cflx_device_count(int* count);

/* ---- process grid (replaces MPI_COMM_WORLD + MPI_Cart_create/sub) ------------------------------------ */
/* rank 0 creates an id and ships it to the other ranks by any host channel (MPI, torch.distributed, a file) */
int cflx_get_unique_id(void* id_out /* CFLX_UNIQUE_ID_BYTES */);
/* COLLECTIVE.  world_size == 1 needs no id (may be NULL).  device = CUDA ordinal this rank drives. */
int cflx_comm_create(int world_size, int world_rank, const void* unique_id, int device, cflx_comm** out);
int cflx_comm_barrier(cflx_comm*); /* COLLECTIVE: device-side barrier + host synchronisation */
void cflx_comm_destroy(cflx_comm*);

/* page-locked host staging buffers for cflx_lu_set_local (cudaHostAlloc / cudaFreeHost) */
int cflx_host_alloc(size_t bytes, void** out);
int cflx_host_free(void* p);

/* ---- sizes (pure host arithmetic, no device needed) ---------------------------------------------------- */
/* lu_params::get_p_grid for a square matrix: P = 1 -> 1x1x1, 2 -> 1x1x2, 4 -> 2x2x1, 8 -> 2x2x2, ... */
int cflx_auto_grid(int M, int N, int P, int* Px, int* Py, int* Pz);
/* dims_out[8] = {M, N, Ml, Nl, Nt, nlayr, Mt, P} after padding, exactly as lu_params::initialize */
int cflx_lu_dims(int M, int N, int v, int Px, int Py, int Pz, int* dims_out);
/* lu_params::InitMatrix, random branch: fills the Ml x Nl row-major local array of `rank` (layers pk != 0 zero) */
int cflx_init_matrix_host(int M, int N, int v, int Px, int Py, int Pz, int rank, int seed, double* local_out);
/* The multipliers of cflx_lu_rbt's random butterflies U (u_out) and V (v_out), depth x M doubles each (row l = level l),
 * either may be NULL: r = exp((w - 0.5) / 10) with the host C library's exp, w = (z >> 11) 2^-53, z = splitmix64's
 * finaliser of seed + 0x9E3779B97F4A7C15 (((2 l + side) << 32) + i + 1) mod 2^64 (side 0 for U, 1 for V); every r lies in
 * [e^-0.05, e^0.05].  CFLX_ERR_ARG for depth outside [1, 4], M < 1, M % 2^depth != 0, or both outputs NULL. */
int cflx_rbt_multipliers(int M, int depth, uint64_t seed, double* u_out, double* v_out);

/* ---- the factorisation ----------------------------------------------------------------------------------- */
/* COLLECTIVE.  Px <= 0 selects cflx_auto_grid(world_size).  Requires Px == Py, Px*Py*Pz == world_size,
 * v % 4 == 0, (v / Pz) % 4 == 0.  Allocates all device memory of the plan. */
int cflx_lu_create(cflx_comm*, int M, int N, int v, int Px, int Py, int Pz, cflx_lu** out);
/* info_out[16] = {M, N, Ml, Nl, Nt, nlayr, P, Px, Py, Pz, pi, pj, pk, rank, v, 0} */
int cflx_lu_info(const cflx_lu*, int* info_out);
/* host -> device copy of this rank's local matrix (conflux tile layout, row-major, ld = Nl); kept pristine */
int cflx_lu_set_local(cflx_lu*, const double* host_local);
/* Input streaming for back-to-back factorisations (no counterpart in the reference, whose input already sits in host
 * memory): the NEXT cflx_lu_factor uploads `host_next` (page-locked; free again when that call returns) into the input
 * buffer behind its own working copy, on a copy stream, so the transfer overlaps the factorisation; the factorisation
 * after that consumes it without a cflx_lu_set_local.  cflx_lu_validate of a run whose input buffer was handed on is
 * refused (CFLX_ERR_STATE). */
int cflx_lu_queue_next_local(cflx_lu*, const double* host_next);
/* COLLECTIVE.  Runs steps 0..Nt-1 on the GPU(s).  ms_out = device time of the main loop only (CUDA events on
 * this rank's stream, after a grid barrier) -- the region the reference times (conflux_opt.hpp:531-532,1805). */
int cflx_lu_factor(cflx_lu*, double* ms_out);
/* COLLECTIVE.  LU of the input with a prescribed row order: P A = L U with the P of `perm`, no pivot search (MAGMA's
 * dgetrf_nopiv on a permuted matrix; static pivoting when tiny > 0).  perm: M ints (M the padded size), row q of P A is
 * row perm[q] of A, the convention of cflx_lu_get_permutation; the same on every rank.  perm = NULL takes the
 * permutation of the last completed factorisation of this handle (pivoted or fixed), which cflx_lu_set_local,
 * cflx_lu_queue_next_local and cflx_lu_equilibrate* keep: a new matrix with the old pivots.  tiny (>= 0, absolute): a
 * pivot u with |u| < tiny becomes copysign(tiny, u), +tiny for +-0; nrepl_out (may be NULL) counts the replacements over
 * the grid.  info_out: 1 + the global column of the first exactly zero pivot (only with tiny = 0), else 0; the
 * factorisation still completes, and entries computed from a zero pivot may be inf or NaN.  nrepl and info are the same
 * on every rank.  ms_out, the input streaming, the scaling the factors carry, and every later call on the factors
 * (solves, rcond, refinement, svx, inverse, det, validate, get_permutation = perm) as cflx_lu_factor.  CFLX_ERR_ARG for
 * tiny < 0 or NaN, a perm that is not a permutation of [0, M), a NULL info_out, or perm differing between ranks (found
 * by one world all-reduce before the first step: every rank returns the error); CFLX_ERR_STATE before cflx_lu_set_local
 * and for perm = NULL before any factorisation completed. */
int cflx_lu_factor_fixed(cflx_lu*, const int* perm, double tiny, int* nrepl_out, int* info_out, double* ms_out);
/* COLLECTIVE.  Random butterfly transform of the input the device holds (MAGMA's dgesv_rbt; Baboulin, Dongarra,
 * Herrmann and Tomov, ACM TOMS 39(2), 2013): A <- W = U^T A V in place, with U and V random recursive butterflies of
 * depth 1 .. 4 (2 in practice) from the multipliers of cflx_rbt_multipliers(M, depth, seed) (u_out / v_out, may be NULL,
 * as there).  With probability one W needs no pivoting: factor it with cflx_lu_factor_fixed in the identity order, then
 * solve with cflx_lu_rbt_solve or cflx_lu_rbt_apply_local.  Each rank transforms its own share, with no communication
 * beyond one world all-reduce that first checks every rank's depth and seed.  Every later call on the factors (solves,
 * rcond, refinement, svx, inverse, det, validate) refers to W, as after an equilibration.  The factors and the solve
 * cache are dropped, as by cflx_lu_set_local; the next factorisation's factors carry the transform.  An input from
 * cflx_lu_set_local or a queued upload carries none.  CFLX_ERR_ARG for depth outside [1, 4], or ranks that differ in
 * depth or seed or refused their arguments (every rank returns the error); CFLX_ERR_UNSUPPORTED when M is not a multiple
 * of 2^depth v Px (the message names the smallest M that works: pad A with the identity); CFLX_ERR_STATE before
 * cflx_lu_set_local, on an input that is already transformed, and on a scaled input (cflx_lu_equilibrate*, apply = 1,
 * which in turn refuses a transformed input). */
int cflx_lu_rbt(cflx_lu*, int depth, uint64_t seed, double* u_out, double* v_out);
/* COLLECTIVE.  Solves A X = B (trans 0) or A^T X = B (trans 1) with factors that carry a transform (cflx_lu_rbt, then a
 * factorisation): X = V inv(W) U^T B, or X = U inv(W)^T V^T B.  B, X, ldb, ldx as cflx_lu_refine.  refine = 1 refines the
 * solution of the transformed system W Y = U^T B (W^T Y = V^T B) as cflx_lu_refine does, so ferr_out and berr_out (nrhs
 * each, may be NULL; not written with refine = 0) are the forward and backward errors of Y in that system, not of X in
 * A X = B.  No singularity check (like getrs).  CFLX_ERR_ARG as cflx_lu_refine, and for refine not 0 / 1; CFLX_ERR_STATE
 * as cflx_lu_solve (with refine = 1 as cflx_lu_refine), and when the factors carry no transform.  Results identical on
 * every rank; leaves the factors, the input, later solves and the launch count as they are. */
int cflx_lu_rbt_solve(cflx_lu*, int trans, int nrhs, const double* B, int ldb, double* X, int ldx, int refine,
                      double* ferr_out, double* berr_out);
/* Not collective.  One butterfly of the factors' transform on the rows of this rank's right-hand side share, in place:
 * op 0 U^T, 1 V, 2 V^T, 3 U.  B_local: the share of cflx_lu_solve_local's layout, Ml x cflx_rhs_local_cols(nrhs, v, Py),
 * leading dimension ldb, host or device memory as there; columns whose global index is >= nrhs are left as they are.
 * A X = B with B and X distributed is apply_local(0) on B, cflx_lu_solve_local, apply_local(1) on X; A^T X = B is
 * apply_local(2), the transposed solve, apply_local(3).  CFLX_ERR_ARG for op outside [0, 3], nrhs < 1, a NULL B_local,
 * ldb below the local column count, or device memory of another device; CFLX_ERR_STATE as cflx_lu_solve, and when the
 * factors carry no transform. */
int cflx_lu_rbt_apply_local(cflx_lu*, int op, int nrhs, double* B_local, int ldb);
/* COLLECTIVE.  C_host (Ml x Nl, may be NULL on layers pk != 0): L\U of P*A in the conflux layout, row
 * (k/Px)*v + i of rank (k%Px, pj, 0) = pivoted row k*v + i; permutation_out[M] = pivotIndsBuff. */
int cflx_lu_get_factors(cflx_lu*, double* C_host, int* permutation_out);
/* device -> host copy of the permutation only (the cheap "result" of a run) */
int cflx_lu_get_permutation(cflx_lu*, int* permutation_out);
/* COLLECTIVE.  The reference's validation (examples/conflux_miniapp.cpp:349-500: L = unit-lower(C), U = upper(C),
 * P from the pivots, P*A - L*U with pdgemm on the Px x Py grid, Frobenius norm reduced over the grid) on the GPU grid:
 * frob_abs_out = ||P*A - L*U||_F (what the reference prints), frob_rel_out = that / ||A||_F.  Either may be NULL.
 * Uses the library's own GEMM and NCCL; allocates ~4 local matrices temporarily; identical result on every rank. */
int cflx_lu_validate(cflx_lu*, double* frob_abs_out, double* frob_rel_out);
/* COLLECTIVE.  = cflx_lu_validate(lu, NULL, rel_out) */
int cflx_lu_residual(cflx_lu*, double* rel_out);
/* COLLECTIVE.  Solves A X = B with the factors of the last cflx_lu_factor (P A = L U), on the GPU grid.
 * B: M x nrhs row-major host array (M = the padded size, info_out[0]), leading dimension ldb >= nrhs, the same on every
 * rank.  X: M x nrhs row-major, ldx >= nrhs, may be NULL on any rank (ldx is then not read); the result is identical on
 * every rank.  The first call after a factorisation prepares and caches per-rank solve data; cflx_lu_set_local /
 * cflx_lu_factor drop it.  Does not modify the factors or the input.  No singularity check (like getrs).
 * CFLX_ERR_ARG for nrhs < 1, a NULL B, ldb < nrhs, or ldx < nrhs with X set; CFLX_ERR_STATE before cflx_lu_factor and
 * after cflx_lu_set_local. */
int cflx_lu_solve(cflx_lu*, int nrhs, const double* B, int ldb, double* X, int ldx);
/* COLLECTIVE.  Solves A^T X = B with the factors of the last cflx_lu_factor, on the GPU grid, like LAPACK's getrs with
 * TRANS = 'T'.  Arguments (ldx is not read when X is NULL), refusals, state rules and caching as cflx_lu_solve. */
int cflx_lu_solve_trans(cflx_lu*, int nrhs, const double* B, int ldb, double* X, int ldx);
/* Pure host.  cols_out: the local columns of an M x nrhs right-hand side share (cflx_lu_solve_local,
 * cflx_chol_solve_local) on any rank of a grid with Py grid columns, v * ceil(ceil(nrhs / v) / Py): lu_params' padding
 * rule applied to nrhs, so nrhs = M gives the matrix's Nl.  CFLX_ERR_ARG for nrhs, v or Py < 1 or a NULL cols_out. */
int cflx_rhs_local_cols(int nrhs, int v, int Py, int* cols_out);
/* COLLECTIVE.  Solves A X = B (trans 0) or A^T X = B (trans 1) with the factors of the last cflx_lu_factor, like
 * ScaLAPACK's pdgetrs, with B and X distributed like A: M x nrhs matrices (M the padded size) tiled v x v, global tile
 * (I, J) on grid position (I % Px, J % Py) at local tile (I / Px, J / Py) of this rank's row-major share of Ml x
 * cflx_rhs_local_cols(nrhs, v, Py), leading dimensions ldb / ldx.  With nrhs = M a share has the shape of A's share.
 * Local columns whose global index is >= nrhs, and the ld padding, are neither read (B) nor written (X).  Shares may be
 * in host or device memory; device memory must be on this rank's device; a host share goes through one temporary device
 * share.  B_local is read on layer pk == 0 only and may be NULL on layers pk != 0; X_local may be NULL on any rank; every
 * layer receives the bits of layer 0.  X_local == B_local (the same host or device pointer) solves in place and needs
 * ldx == ldb; shares that overlap otherwise are not allowed.  The columns are solved in blocks of the width of
 * cflx_lu_inverse, each assembled on the device and computed exactly as cflx_lu_solve (or cflx_lu_solve_trans) computes
 * those columns alone, so device memory is bounded by one block whatever nrhs is.  The matrix solved is the one the
 * factors represent (the scaled one after cflx_lu_equilibrate), as for cflx_lu_solve.  No singularity check (like getrs).
 * CFLX_ERR_ARG for trans not 0 / 1, nrhs < 1, ldb (layer 0) or ldx (X set) below the local column count, a NULL B_local
 * on layer 0, X_local == B_local with ldx != ldb, or device memory of another device.  CFLX_ERR_STATE as cflx_lu_solve.
 * Every rank passes the same trans and nrhs.  Leaves the factors, the permutation, the input, the scaling record, later
 * solves and the launch count as they are. */
int cflx_lu_solve_local(cflx_lu*, int trans, int nrhs, const double* B_local, int ldb, double* X_local, int ldx);
/* COLLECTIVE.  LAPACK dgecon (NORM = '1') on the GPU grid: rcond_out = 1 / (||A||_1 ||inv(A)||_1) with ||inv(A)||_1
 * estimated by Hager-Higham's method (dlacn2: at most 5 iterations, a few solves with one right-hand side), anorm_out
 * (may be NULL) = ||A||_1 of the padded M x M input.  rcond is 0 when ||A||_1 is 0 or the estimate is not finite (an
 * exactly singular U), with CFLX_OK.  Identical on every rank.  CFLX_ERR_STATE as cflx_lu_solve, and when the input
 * buffer of the last run was handed to the queued next matrix.  Leaves the factors, the permutation and any later solve
 * as they are. */
int cflx_lu_rcond(cflx_lu*, double* rcond_out, double* anorm_out);
/* COLLECTIVE.  LAPACK dgerfs on the GPU grid with the factors of the last cflx_lu_factor and the input it kept:
 * trans 0: A X = B, 1: A^T X = B.  B, X: M x nrhs row-major host arrays (M = the padded size), ldb / ldx >= nrhs, the same
 * on every rank; X holds a solution on entry (e.g. from cflx_lu_solve) and the refined one on return, identical on
 * every rank.  ferr_out / berr_out: nrhs doubles each, either may be NULL; with ferr_out NULL the estimator does not run.
 * Per column, as dgerfs: at most 5 corrections while the componentwise backward error berr = max_i |b - op(A) x|_i /
 * (|op(A)| |x| + |b|)_i exceeds 2^-53 and at least halves; ferr bounds ||x - x_true||_inf / ||x||_inf by the Hager-Higham
 * estimate of || |inv(op A)| (|r| + (M + 1) 2^-53 (|op(A)| |x| + |b|)) ||_inf.  CFLX_ERR_ARG for trans not 0 / 1, nrhs < 1,
 * ldb or ldx < nrhs, a NULL B or X; CFLX_ERR_STATE as cflx_lu_rcond.  No singularity check (like dgerfs).  Leaves the
 * factors, the permutation, the input, later solves and the launch count as they are. */
int cflx_lu_refine(cflx_lu*, int trans, int nrhs, const double* B, int ldb, double* X, int ldx, double* ferr_out,
                   double* berr_out);
/* COLLECTIVE.  LAPACK dgerfsx on the GPU grid: refinement with the residual b - op(A)(y + y_tail) in double-double,
 * converging to full working accuracy whenever cond * 2^-53 is safely below 1, with error bounds and a trust flag per
 * right-hand side.  trans, B, X, ldb, ldx and the state rules as cflx_lu_refine; the matrix is the one the factors
 * represent (the scaled A_s after cflx_lu_equilibrate).  rcond_out (may be NULL): dgecon of A_s in the infinity-norm
 * (trans 0) or the 1-norm (trans 1).  berr_out (nrhs, may be NULL): max_i (|r_i| + (M + 1) safmin) / (|op(A_s)| |y| +
 * |b|)_i.  err_bnds_norm_out / err_bnds_comp_out: nrhs x 3 row-major, row j = {trust, err, rcond} of column j (LAPACK's
 * ERR_BNDS(j, 1..3)), bounding ||x - x_true||_inf / ||x||_inf and max_i |x_i - x_true,i| / |x_i| of the unscaled
 * x = diag(d) y (d: c for trans 0 with equed C / B, r for trans 1 with equed R / B, else ones); err_bnds_comp_out NULL:
 * componentwise convergence is neither pursued nor estimated.  info_out: k for the first exactly zero U(k,k) (X left as
 * it was, rcond 0, nothing else written); M + j for the first column j whose bound was set to 1 because its condition
 * estimate is below M 2^-53; 0 otherwise.  CFLX_ERR_ARG as cflx_lu_refine and for a NULL err_bnds_norm_out or info_out;
 * CFLX_ERR_STATE as cflx_lu_rcond.  Results identical on every rank; leaves the factors, the permutation, the input,
 * later solves and the launch count as they are. */
int cflx_lu_refine_x(cflx_lu*, int trans, int nrhs, const double* B, int ldb, double* X, int ldx, double* rcond_out,
                     double* berr_out, double* err_bnds_norm_out, double* err_bnds_comp_out, int* info_out);
/* COLLECTIVE.  LAPACK dgeequ on the input the device holds (the padded M x M matrix of cflx_lu_set_local), and with
 * apply = 1 dlaqge: the input is scaled in place, a_ij = (c_j r_i) a_ij (only r or only c for equed 'R' / 'C'), when
 * rowcnd < 0.1, colcnd < 0.1 or amax is outside [dlamch('S') / dlamch('P'), its reciprocal].  r_out / c_out (M doubles,
 * may be NULL): the row and column scales; rowcnd_out, colcnd_out, amax_out (may be NULL) as dgeequ; equed_out (may be
 * NULL): 'N', 'R', 'C' or 'B' ('N' when apply = 0).  info_out: 0, i for the first zero row i, M + j for the first zero
 * column j (1-based; the scales are then not applied, and r_out holds the row maxima as dgeequ leaves them).  The
 * factorisation and the solve cache are dropped, as by cflx_lu_set_local; the next cflx_lu_factor factors the scaled
 * matrix and its factors carry the scaling to cflx_lu_svx; cflx_lu_validate, _rcond and _refine then refer to the scaled
 * matrix.  An input from cflx_lu_set_local or a queued upload carries no scaling; apply = 0 on an input that is already
 * scaled is a query of the scaled matrix and leaves the scaling it carries as it was.  Identical results on every rank.
 * CFLX_ERR_ARG for apply not 0 / 1 or a NULL info_out; CFLX_ERR_STATE before cflx_lu_set_local, and for apply = 1 on an
 * input that is already scaled. */
int cflx_lu_equilibrate(cflx_lu*, int apply, double* r_out, double* c_out, double* rowcnd_out, double* colcnd_out,
                        double* amax_out, char* equed_out, int* info_out);
/* COLLECTIVE.  LAPACK dgesvx after the factorisation (FACT = 'F' on this library's factors, with the scaling they carry
 * from cflx_lu_equilibrate): trans 0: A X = B, 1: A^T X = B.  B is scaled by r (trans 0, equed R / B) or c (trans 1,
 * equed C / B); rpvgrw_out (may be NULL) = max |A_s| / max |triu(U)|, or 1 when the latter is 0; rcond_out = dgecon of the
 * scaled matrix in the 1-norm (trans 0, the bits of cflx_lu_rcond) or the infinity-norm (trans 1); X is solved, refined
 * as cflx_lu_refine refines it (ferr_out / berr_out, nrhs doubles each, may be NULL), and unscaled by c (trans 0) or r
 * (trans 1), ferr divided by colcnd or rowcnd.  equed_out (may be NULL): the factors' scaling.  info_out: k when U(k,k)
 * is exactly zero (the first such k; rcond = 0, rpvgrw over the leading k columns, X not written); M + 1 when rcond <
 * 2^-53 (X is still computed); 0 otherwise.  B, X, ldb, ldx as cflx_lu_refine; results identical on every rank.
 * CFLX_ERR_ARG as cflx_lu_refine and for a NULL rcond_out or info_out; CFLX_ERR_STATE as cflx_lu_rcond. */
int cflx_lu_svx(cflx_lu*, int trans, int nrhs, const double* B, int ldb, double* X, int ldx, double* rcond_out,
                double* ferr_out, double* berr_out, double* rpvgrw_out, char* equed_out, int* info_out);
/* COLLECTIVE.  LAPACK dgeequb (+ dlaqge when apply): cflx_lu_equilibrate with the scales rounded to powers of two.  The
 * row maxima are rounded to 2^INT(log(x) / log(2)) before rcmin, rcmax and amax are taken, then the column maxima of
 * |a| r likewise; the exponents come from the host's log, as LAPACK's.  r_out / c_out hold the rounded maxima on the
 * info paths.  Scaling A, scaling B and unscaling X are then exact (barring underflow), so the factors of the scaled
 * matrix are those of diag(r) A diag(c) and cflx_lu_svxx's bounds carry over to the unscaled solution.  Arguments,
 * state rules and the scaling record as cflx_lu_equilibrate. */
int cflx_lu_equilibrate_b(cflx_lu*, int apply, double* r_out, double* c_out, double* rowcnd_out, double* colcnd_out,
                          double* amax_out, char* equed_out, int* info_out);
/* COLLECTIVE.  LAPACK dgesvxx after the factorisation (FACT = 'F' on this library's factors, with the scaling they carry
 * from cflx_lu_equilibrate_b, cflx_lu_equilibrate or none): trans 0: A X = B, 1: A^T X = B.  rpvgrw_out (may be NULL):
 * dla_gerpvgrw, the minimum of 1 and of max_i |a_ij| / max_{i <= j} |u_ij| over the columns j with a non-zero
 * denominator.  B is scaled by r (trans 0, equed R / B) or c (trans 1, equed C / B), solved, refined as
 * cflx_lu_refine_x refines it (rcond_out, berr_out, err_bnds_norm_out and err_bnds_comp_out as there, the bounds for
 * the unscaled solution, so nothing is divided by colcnd), and X is unscaled by c (trans 0) or r (trans 1).  equed_out
 * (may be NULL): the factors' scaling.  info_out: k for the first exactly zero U(k,k) (rpvgrw over the leading k columns,
 * rcond 0, nothing else written, X left as it was); M + j from the refinement as cflx_lu_refine_x (there is no
 * dgesvx-style M + 1); 0 otherwise.  CFLX_ERR_ARG as cflx_lu_refine_x and for a NULL rcond_out; CFLX_ERR_STATE as
 * cflx_lu_rcond.  Results identical on every rank; leaves the factors, the permutation, the input, the scaling record,
 * later solves and the launch count as they are. */
int cflx_lu_svxx(cflx_lu*, int trans, int nrhs, const double* B, int ldb, double* X, int ldx, double* rcond_out,
                 double* rpvgrw_out, double* berr_out, double* err_bnds_norm_out, double* err_bnds_comp_out,
                 char* equed_out, int* info_out);
/* COLLECTIVE.  inv(A) of the padded M x M matrix factored by the last cflx_lu_factor (P A = L U), on the GPU grid, like
 * LAPACK's dgetri.  Ainv_local: Ml x Nl row-major, the conflux layout of cflx_lu_set_local; host or device memory; may be
 * NULL on any rank.  Every rank receives the share of its grid position (pi, pj); layers pk != 0 receive the bits of
 * layer 0.  info_out: k when U(k,k) is exactly zero (the first such k, counted from 1; nothing is written); 0 otherwise.
 * When the factors carry a scaling (cflx_lu_equilibrate), this is the inverse of the scaled matrix, as for
 * cflx_lu_validate / _rcond.  The columns come from solves A X = I, so the right residual A X - I is small (dgetri bounds
 * the left one, X A - I).  CFLX_ERR_ARG for a NULL info_out.  CFLX_ERR_STATE as cflx_lu_solve.  Leaves the factors, the
 * permutation, the input, later solves and the launch count as they are. */
int cflx_lu_inverse(cflx_lu*, double* Ainv_local, int* info_out);
/* COLLECTIVE.  det of the matrix factored by the last cflx_lu_factor (P A = L U), det = sign mant 2^exp, without overflow
 * or underflow: sign_out (+1, -1, 0), logabsdet_out (log |det|; -inf when singular), mant_out / exp_out (the exact-range
 * det: |det| = mant 2^exp, mant in [0.5, 1), or 0 when singular), info_out (k for the first exactly zero U(k,k), counted
 * from 1, else 0).  Any output may be NULL except info_out.  This is the determinant of the padded M x M matrix, as
 * cflx_lu_rcond's anorm is its norm: a caller who pads with the identity gets det(A).  A U(k,k) that is inf or NaN with no
 * zero before it gives sign, mant and logabsdet NaN.  unscaled = 0: the matrix the factors represent (the scaled one after
 * cflx_lu_equilibrate, as cflx_lu_rcond / _inverse); 1: divided by the scales the factors carry (prod(r) for equed 'R',
 * prod(c) for 'C', both for 'B'), i.e. det of the input before equilibration (the same bits as 0 when equed = 'N').
 * Identical bits on every rank and on every call.  CFLX_ERR_ARG for unscaled not 0 / 1 or a NULL info_out;
 * CFLX_ERR_STATE as cflx_lu_solve.  Leaves the factors, the permutation, the input, later solves and the launch count as
 * they are. */
int cflx_lu_det(cflx_lu*, int unscaled, double* sign_out, double* logabsdet_out, double* mant_out, int64_t* exp_out,
                int* info_out);
/* 1 when this plan's trailing update runs on the int8 wgmma digit-plane path (ozaki.cu), 0 for the FP64 DMMA kernel
 * (gemm.cu) */
int cflx_lu_uses_ozaki(const cflx_lu*);
/* number of kernels this plan launched since the last call (for bench.py's gpu_launches) */
int cflx_lu_launch_count(cflx_lu*, int64_t* count_out, int reset);
/* per-phase device time of the last cflx_lu_factor when profiling was enabled: ms_out[8] =
 * {panel, tournament+bcast, row moves, reduce+gather, trsm, gemm, stores, other} */
/* mode 0 off; 1 serialising timers (per-phase device time without overlap); 2 non-serialising timeline: CUDA event
 * pairs on the launching streams, resolved after the run -- the timeline of the real, overlapped execution.  Every region
 * is also an NVTX range named like the reference's semiprof regions (src/conflux/lu/profiler.hpp:5-19: step0_copy,
 * step1_lup, step2_pushingpivots, step4_dtrsm, step6_dgemm, ...). */
int cflx_lu_set_profiling(cflx_lu*, int mode);
int cflx_lu_phase_ms(cflx_lu*, double* ms_out);
/* JSON text {"main": {"step6_dgemm": [ms, count], ...}, "side": {...}} of the last profiled cflx_lu_factor (main stream /
 * look-ahead stream).  Returns 0, or the buffer length needed when buf is NULL or too small. */
int cflx_lu_timeline(cflx_lu*, char* buf, int buf_len);
/* CUDA-event timing of the dominant kernel (the trailing-update DGEMM launches of the last cflx_lu_factor, events
 * recorded on the launching stream): summed device ms and the algorithmic flops 2*m*n*k of those launches */
int cflx_lu_set_kernel_timing(cflx_lu*, int enabled);
int cflx_lu_trailing_stats(cflx_lu*, double* ms_out, double* flops_out);
void cflx_lu_destroy(cflx_lu*);

/* ---- CONFCHOX: Cholesky factorisation A = L L^T (lower) on the same process grid (BASELINE config C5) -----------------
 * Reference interfaces replaced (src/conflux/cholesky):
 *   initialize(argc, argv, N, v, grid)  Cholesky.cpp:60-160 (grid / tile choice :75-134)  -> cflx_chol_auto_grid/_tile, cflx_chol_create
 *   CholeskyIO::generateInputMatrixDistributed  CholeskyIO.cpp:100-172                   -> cflx_chol_init_matrix_host
 *   parallelCholesky()                  Cholesky.cpp:760-921                              -> cflx_chol_factor
 *   finalize(clean)                     Cholesky.cpp:160-175                              -> cflx_chol_destroy
 * Local data: row-major Ml x Nl, tile (gi, gj) of the v x v tiling on rank (gi % Px, gj % Py) at local tile (gi / Px,
 * gj / Py); ranks are numbered (pi * Py + pj) * Pz + pk like the LU path; only the lower triangle is referenced. */
typedef struct cflx_chol cflx_chol;
int cflx_chol_auto_grid(int P, int N, int* grid3_out);
int cflx_chol_auto_tile(int N, int P, int Pz);
/* dims_out[6] = {N padded to a multiple of v, Kappa (tiles per dimension), Ml, Nl, v / Pz, P} */
int cflx_chol_dims(int N, int v, int Px, int Py, int Pz, int* dims_out);
int cflx_chol_init_matrix_host(int N, int v, int Px, int Py, int Pz, int rank, double* local_out);
/* COLLECTIVE.  Px <= 0 / v <= 0 select the reference's automatic choices.  Requires v % 4 == 0, (v / Pz) % 4 == 0, v <= 512. */
int cflx_chol_create(cflx_comm*, int N, int v, int Px, int Py, int Pz, cflx_chol** out);
/* info_out[16] = {N, v, Kappa, Ml, Nl, v / Pz, P, Px, Py, Pz, pi, pj, pk, rank, 0, 0} */
int cflx_chol_info(const cflx_chol*, int* info_out);
int cflx_chol_set_local(cflx_chol*, const double* host_local);
/* COLLECTIVE.  ms_out = device time of the factorisation loop (the region the reference's miniapp times). */
int cflx_chol_factor(cflx_chol*, double* ms_out);
int cflx_chol_get_local(cflx_chol*, double* L_host);
/* COLLECTIVE.  ||A - L L^T||_F over the lower triangle, absolute and relative to ||A||_F, computed on the GPU grid. */
int cflx_chol_validate(cflx_chol*, double* frob_abs_out, double* frob_rel_out);
/* COLLECTIVE.  Solves A X = B with the factor of the last successful cflx_chol_factor (A = L L^T), on the GPU grid, like
 * LAPACK's potrs.  B: N x nrhs row-major host array (N = the padded size, info_out[0]), leading dimension ldb >= nrhs, the
 * same on every rank.  X: N x nrhs row-major, ldx >= nrhs, may be NULL on any rank; the result is identical on every rank.
 * CFLX_ERR_ARG for nrhs < 1, ldb < nrhs, ldx < nrhs with X set, or a NULL B.  CFLX_ERR_STATE before a successful
 * cflx_chol_factor, after cflx_chol_set_local, and after a factorisation that found a non-positive pivot.  The first call
 * after a factorisation prepares and caches per-rank solve data; cflx_chol_set_local / cflx_chol_factor drop it.  Does not
 * modify the factor or the input. */
int cflx_chol_solve(cflx_chol*, int nrhs, const double* B, int ldb, double* X, int ldx);
/* COLLECTIVE.  Solves A X = B with the factor of the last successful cflx_chol_factor, like ScaLAPACK's pdpotrs, with B
 * and X distributed like A: the layout, memory, layer, in-place and block rules of cflx_lu_solve_local, each block
 * computed exactly as cflx_chol_solve computes those columns alone.  Only the rows of real tiles (global tile index <
 * Kappa) are read or written.  The matrix solved is the scaled one after cflx_chol_equilibrate, as for cflx_chol_solve.
 * CFLX_ERR_ARG as cflx_lu_solve_local (without trans); CFLX_ERR_STATE as cflx_chol_solve.  Every rank passes the same
 * nrhs.  Side effects as cflx_lu_solve_local. */
int cflx_chol_solve_local(cflx_chol*, int nrhs, const double* B_local, int ldb, double* X_local, int ldx);
/* COLLECTIVE.  LAPACK dpocon on the GPU grid: rcond_out = 1 / (||A||_1 ||inv(A)||_1), ||A||_1 of the symmetric input
 * whose lower triangle is stored (anorm_out, may be NULL), ||inv(A)||_1 estimated by Hager-Higham's method with solves.
 * Identical on every rank.  CFLX_ERR_STATE as cflx_chol_solve.  Leaves the factor and any later solve as they are. */
int cflx_chol_rcond(cflx_chol*, double* rcond_out, double* anorm_out);
/* COLLECTIVE.  LAPACK dporfs (UPLO = 'L') with the factor of the last successful cflx_chol_factor and the input it kept
 * (its lower triangle); the arguments and results of cflx_lu_refine without trans.  CFLX_ERR_STATE as cflx_chol_solve. */
int cflx_chol_refine(cflx_chol*, int nrhs, const double* B, int ldb, double* X, int ldx, double* ferr_out,
                     double* berr_out);
/* COLLECTIVE.  LAPACK dporfsx (UPLO = 'L'): cflx_lu_refine_x without trans, with the symmetric residual from the stored
 * lower triangle, rcond_out = dpocon, and d = s for equed Y.  info_out: M + j as cflx_lu_refine_x, else 0.
 * CFLX_ERR_STATE as cflx_chol_solve. */
int cflx_chol_refine_x(cflx_chol*, int nrhs, const double* B, int ldb, double* X, int ldx, double* rcond_out,
                       double* berr_out, double* err_bnds_norm_out, double* err_bnds_comp_out, int* info_out);
/* COLLECTIVE.  LAPACK dpoequ on the input the device holds, and with apply = 1 dlaqsy (UPLO = 'L'): s_i = 1 / sqrt(a_ii),
 * scond = sqrt(min a_ii) / sqrt(max a_ii), amax = max a_ii; the stored lower triangle of the real tiles is scaled in
 * place, a_ij = (s_j s_i) a_ij, when scond < 0.1 or amax is outside [dlamch('S') / dlamch('P'), its reciprocal].
 * s_out (N doubles), scond_out, amax_out, equed_out ('N' or 'Y') may be NULL.  info_out: i for the first a_ii <= 0
 * (1-based; s_out then holds the diagonal and nothing is scaled), else 0.  State rules and the scaling record as
 * cflx_lu_equilibrate. */
int cflx_chol_equilibrate(cflx_chol*, int apply, double* s_out, double* scond_out, double* amax_out, char* equed_out,
                          int* info_out);
/* COLLECTIVE.  LAPACK dposvx after a successful factorisation, with the scaling the factor carries: B scaled by s,
 * rcond_out = dpocon of the scaled matrix (the bits of cflx_chol_rcond), X solved, refined as cflx_chol_refine refines it
 * and unscaled by s, ferr divided by scond.  info_out: N + 1 when rcond < 2^-53 (X is still computed), else 0.
 * Arguments as cflx_chol_refine; CFLX_ERR_ARG also for a NULL rcond_out or info_out; CFLX_ERR_STATE as cflx_chol_solve. */
int cflx_chol_svx(cflx_chol*, int nrhs, const double* B, int ldb, double* X, int ldx, double* rcond_out, double* ferr_out,
                  double* berr_out, char* equed_out, int* info_out);
/* COLLECTIVE.  LAPACK dpoequb (+ dlaqsy when apply): cflx_chol_equilibrate with s_i = 2^INT((-0.5 / log(2)) log(a_ii)),
 * the exponents from the host's log, as LAPACK's; scond, amax, info and s_out on the info path as dpoequ.  Arguments,
 * state rules and the scaling record as cflx_chol_equilibrate. */
int cflx_chol_equilibrate_b(cflx_chol*, int apply, double* s_out, double* scond_out, double* amax_out, char* equed_out,
                            int* info_out);
/* COLLECTIVE.  LAPACK dposvxx (UPLO = 'L') after a successful factorisation, with the scaling the factor carries:
 * rpvgrw_out (may be NULL) = dla_porpvgrw, the minimum of 1 and of max |a_ij| / max |l_ij| over the rows i >= j of the
 * stored lower triangles, per column j with a non-zero denominator; rcond_out = dpocon; B scaled by s, solved, refined as
 * cflx_chol_refine_x refines it and unscaled by s.  info_out: N + j from the refinement, else 0.  A factorisation that
 * found a non-positive pivot is refused (CFLX_ERR_STATE), where dposvxx would return info = k.  Arguments, results and
 * side effects otherwise as cflx_lu_svxx without trans. */
int cflx_chol_svxx(cflx_chol*, int nrhs, const double* B, int ldb, double* X, int ldx, double* rcond_out,
                   double* rpvgrw_out, double* berr_out, double* err_bnds_norm_out, double* err_bnds_comp_out,
                   char* equed_out, int* info_out);
/* COLLECTIVE.  inv(A) from the factor of the last successful cflx_chol_factor (A = L L^T), like LAPACK's dpotri
 * (UPLO = 'L'): the real tiles on and below the diagonal of this rank's Ml x Nl share hold inv(A), whole diagonal tiles
 * included.  The tiles above the diagonal and the local tiles with a global index >= Kappa are zero.  Host or device
 * memory; may be NULL.  Every layer receives the bits of layer 0.  As for cflx_lu_inverse, the right residual is the
 * small one.  CFLX_ERR_STATE as cflx_chol_solve.  Adds nothing to cflx_chol_launch_count. */
int cflx_chol_inverse(cflx_chol*, double* Ainv_local);
/* COLLECTIVE.  det = prod(l_ii)^2 of the padded N x N matrix of the last successful cflx_chol_factor: logdet_out, and the
 * exact-range det mant_out 2^exp_out as cflx_lu_det's; unscaled = 1 divides by prod(s)^2 of the scaling the factor
 * carries (equed 'Y').  Any output may be NULL.  Determinism and side effects as cflx_lu_det; CFLX_ERR_ARG for unscaled
 * not 0 / 1; CFLX_ERR_STATE as cflx_chol_solve. */
int cflx_chol_det(cflx_chol*, int unscaled, double* logdet_out, double* mant_out, int64_t* exp_out);
/* number of kernels this object counted since the last reset (bench.py's gpu_launches); cflx_chol_solve adds none */
int cflx_chol_launch_count(cflx_chol*, int64_t* count_out, int reset);
void cflx_chol_destroy(cflx_chol*);

/* ---- single-device building blocks exposed for tests and micro-benchmarks (host buffers in, host out) ----- */
/* D = beta*C + alpha * AT^T * B on the trailing-update kernel, at a window of whole row-major host buffers, as the
 * factorisation launches it: AT [at_rows x ldat] read from element at_off (K rows of M, rounded up to even), B
 * [b_rows x ldb] from element b_off (K rows of N), C [c_rows x ldc] updated in rows [row_off, row_off + M) x columns
 * [col_off, col_off + N).  in_place != 0: D is C on the device; else D is a device copy of C.  D_out / C_out (optional,
 * c_rows x ldc) receive the whole D and C buffers after the call.  N, K % 4, ldat, ldb, ldc and the offsets (but row_off)
 * even; the window must lie inside the buffers.  ms_out: mean device time of one launch over reps. */
int cflx_dbg_gemm_tn(int M, int N, int K, const double* AT, int at_rows, int64_t ldat, int64_t at_off, const double* B,
                     int b_rows, int64_t ldb, int64_t b_off, const double* C, int c_rows, int64_t ldc, int row_off,
                     int col_off, double alpha, double beta, int in_place, double* D_out, double* C_out, int reps,
                     double* ms_out);
/* D = beta*C + alpha * A * B with A [M x K], B [K x N], C/D [M x N], all row-major, dense: the narrow GEMM of the solve */
int cflx_dbg_gemm_narrow(int M, int N, int K, const double* A, const double* B, const double* C, double alpha, double beta,
                         double* D, int reps, double* ms_out);
/* D = beta*C + alpha * AT^T * B with AT [K x M], B [K x N], C/D [M x N], all row-major, dense: the transposed narrow GEMM
 * of the Cholesky solve.  On the device AT gets an even leading dimension >= M, so any M >= 1 can be run. */
int cflx_dbg_gemm_narrow_tn(int M, int N, int K, const double* AT, const double* B, const double* C, double alpha,
                            double beta, double* D, int reps, double* ms_out);
/* D = beta*C + alpha * op(A) * B on the solve's narrow GEMM (trans == 0: op(A) = A, the block of M rows and K columns of
 * A at row a_row, column a_col; trans != 0: the transposed kernel, op(A) = A^T with A's block K rows of M), at windows
 * of whole row-major host buffers, as the solve engine launches it: A [a_rows x lda], B [b_rows x ldb] read from its
 * block of K rows of N at (b_row, b_col), C [c_rows x ldc] updated in rows [c_row, c_row + M) x columns
 * [c_col, c_col + N).  C is read only when beta != 0.  in_place != 0: D is C on the device; else D is a device copy of
 * C.  D_out / C_out (optional, c_rows x ldc) receive the whole D and C buffers after the call.  Refused: a block or
 * window outside its buffer, K < 0, K % 4 != 0 (trans == 0), an odd lda or a_col (A's rows 16-byte aligned). */
int cflx_dbg_gemm_narrow_window(int trans, int M, int N, int K, const double* A, int a_rows, int64_t lda, int a_row,
                                int a_col, const double* B, int b_rows, int64_t ldb, int b_row, int b_col, const double* C,
                                int c_rows, int64_t ldc, int c_row, int c_col, double alpha, double beta, int in_place,
                                double* D_out, double* C_out);
/* One diagonal tile of the solve engine: the v x v tile at (row0, col0) of the row-major share [rows x ld] (lower != 0:
 * the Cholesky factor L with zeros above its diagonal; 0: the LU's L\U with a unit L), its nb x nb diagonal blocks
 * inverted as the solves cache them, then Y_out = T^-1 R (R and Y_out v x ldn) by the solves' block sweep, with tri
 * 0 .. 4 = T = L (Lower), U (Upper), L^T (LowerT, Cholesky), L^T (UnitLowerT, the LU's unit L), U^T (UpperT).  The
 * Cholesky tile takes Lower or LowerT, the LU tile any but LowerT.  inv_out (optional, 2 v nb) receives the cached
 * blocks: v / nb row-major nb x nb forward blocks (inv(L_jj)), then v / nb backward ones (inv(U_jj), or inv(L_jj)^T of
 * the Cholesky tile).  nb in 4, 8, ..., 128 with v % nb == 0; ld and col0 even; the tile inside the share. */
int cflx_dbg_diag_solve(int tri, int lower, int v, int nb, const double* share, int rows, int64_t ld, int row0, int col0,
                        int ldn, const double* R, double* Y_out, double* inv_out);
/* The share a per-share hook runs on: one rank's row-major Ml x Nl share of a block-cyclic matrix of v x v tiles on a
 * Px x Py grid.  Global tile (I, J) lives on grid position (I % Px, J % Py) at local tile (I / Px, J / Py), so local row
 * r of the share at (pi, pj) is global row ((r / v) Px + pi) v + r % v, and local column c likewise with Py and pj.
 *   M       the global order: M-vectors and M-row buffers are indexed by global row or column;
 *   v       the tile;  Ml, Nl  the share's rows and columns;  Px, Py  the grid;  pi, pj  the share's position on it;
 *   Kappa   the real tiles: global tiles with an index >= Kappa are padding, which the symmetric (Cholesky) passes
 *           neither read nor write.
 * Every hook that takes one refuses v < 1, Px or Py < 1, a position off the grid (pi outside [0, Px), pj outside
 * [0, Py)) and Ml or Nl < 0.  Where a hook says so it also needs the share tiled (Ml and Nl multiples of v), covered
 * (M >= (Ml / v) Px v and M >= (Nl / v) Py v) or non-empty (Ml and Nl >= 1).  A refusal names the condition. */
typedef struct { int M, v, Kappa, Ml, Nl, Px, Py, pi, pj; } cflx_share_layout;
/* the residual kernels of cflx_*_refine on one layer-0 share A (Ml x Nl, M unused; Nl even, v a multiple of 4): mode 0
 * (NN) P = A Xc, Q = |A| |Xc| (Ml rows); 1 (TN) P = A^T Xr, Q = |A|^T |Xr| (Nl rows); 2 the stored lower triangle of the
 * real tiles, NN over global row >= column into rows [0, Ml) and TN over global row > column into rows [Ml, Ml + Nl).
 * Xc: Nl x nrhs, Xr: Ml x nrhs (either may be NULL when the mode does not read it).  P_out / Q_out: nrhs columns.
 * ms_out: mean device time of one launch over reps. */
int cflx_dbg_residual(int mode, const cflx_share_layout* share, const double* A, int nrhs, const double* Xc,
                      const double* Xr, double* P_out, double* Q_out, int reps, double* ms_out);
/* the double-double residual kernels of cflx_*_refine_x, arguments as cflx_dbg_residual but any v: hi_out + lo_out =
 * op(A) (X + X_tail) in mode 0, 1 or 2, from Xc + Xct (NN) or Xr + Xrt (TN); either tail may be NULL (zero). */
int cflx_dbg_residual_x(int mode, const cflx_share_layout* share, const double* A, int nrhs, const double* Xc,
                        const double* Xct, const double* Xr, const double* Xrt, double* hi_out, double* lo_out, int reps,
                        double* ms_out);
/* the per-share kernels of cflx_*_equilibrate and cflx_lu_svx on one layer-0 share A (tiled, covered).  r, c: M-vectors
 * (r is also the Cholesky's s).  Each output may be NULL:
 *   rowmax_out / colmax_out (M): max |a| by global row, max |a| r_i by global column, zeros where the share holds none;
 *   diag_out (M): a_gg on the share's diagonal tiles with a global tile index < Kappa, zeros elsewhere;
 *   scaled_out (Ml x Nl): the share after dlaqge's scaling for equed ('N', 'R', 'C', 'B');
 *   sym_scaled_out (Ml x Nl): the share after dlaqsy's (s_j s_i) a on the real tiles' lower triangle, the rest untouched;
 *   growth_out[2]: {max |a| over global row <= column, max |a|}, both over global columns < ncols (the share read as both
 *   L\U and the input); zero_pivot_out: 1 + the first global g < M on the share's diagonal with a_gg == 0, or 0. */
int cflx_dbg_equil(const cflx_share_layout* share, const double* A, const double* r, const double* c, char equed, int ncols,
                   double* rowmax_out, double* colmax_out, double* diag_out, double* scaled_out, double* sym_scaled_out,
                   double* growth_out, int* zero_pivot_out);
/* the per-column pivot growth pass of cflx_lu_svxx (mode 0), cflx_chol_svxx (mode 1) and cflx_lu_svx on one layer-0
 * share (tiled, covered): F the factor and A the input, both Ml x Nl.  amax_out / fmax_out (M each, may be NULL), by
 * global column j < ncols, zeros elsewhere: mode 0 max |a_ij| over every row and max |f_ij| over the rows i <= j; mode 1
 * both over the real tiles' rows j <= i < ncols.  Nothing outside these masks is read. */
int cflx_dbg_growth_cols(int mode, const cflx_share_layout* share, int ncols, const double* F, const double* A,
                         double* amax_out, double* fmax_out);
/* the per-share kernels of cflx_lu_inverse (mode 0) and cflx_chol_inverse (mode 1) on one share (tiled, covered), for
 * the block of nc columns from global column c0 (c0 + nc <= M).  Each output may be NULL:
 *   W_out (Ml x ldn, ldn = nc rounded up to a multiple of 8): the seed, W[r][j] = (global row of r == c0 + j) for the
 *   first `rows` local rows, zero in the rest;
 *   share_inout (Ml x Nl): column j < nc of X (M x ldx, by global row) scattered into the share, to global column
 *   perm[c0 + j] (mode 0, perm: M ints) or c0 + j (mode 1, real tiles on and below the diagonal only); then, with
 *   zero_fill in mode 1, zeros on every entry that scatter never writes.  Every other entry keeps its value. */
int cflx_dbg_inverse_share(int mode, const cflx_share_layout* share, int c0, int nc, int rows, const double* X, int ldx,
                           const int* perm, double* W_out, double* share_inout, int zero_fill);
/* the pack and scatter kernels of cflx_lu_solve_local (mode 0) and cflx_chol_solve_local (mode 1) on one right-hand side
 * share (tiled; Nl = cflx_rhs_local_cols(nrhs, v, Py); M >= (Ml / v) Px v), for the block of w columns from global
 * column c0 of an M x nrhs matrix (c0 + w <= nrhs).  The rows are every local row (mode 0) or those of real tiles (mode
 * 1).  Each output may be NULL:
 *   Bk_out (M x ldn, ldn = w rounded up to a multiple of 8): the pack of B (Ml x ldb, ldb >= Nl), the share's entries of
 *   the block by global row, zero elsewhere;
 *   X_inout (Ml x ldx, ldx >= Nl): Xk (M x ldn, by global row) scattered into the share's columns of the block.  Every
 *   other entry keeps its value. */
int cflx_dbg_solve_local_share(int mode, const cflx_share_layout* share, int nrhs, int c0, int w, const double* B, int ldb,
                               double* Bk_out, const double* Xk, double* X_inout, int ldx);
/* the per-share pass of cflx_lu_rcond's and cflx_chol_rcond's 1-norm (mode 0: every entry; mode 1: the symmetric matrix
 * stored as the lower triangle of its real tiles) and of the infinity-norm (mode 2) on one layer-0 share A (tiled,
 * covered, non-empty), before the all-reduce over the grid.  out (M doubles): by global index, this share's part of the
 * column sums of |a| (modes 0, 1) or of the row sums (mode 2), zero where it holds nothing. */
int cflx_dbg_norm_share(int mode, const cflx_share_layout* share, const double* A, double* out);
/* cflx_lu_rbt's butterflies on one share (tiled; Ml, and for op 4 Nl, a multiple of 2^depth v), in place: op 0 U^T, 1 V,
 * 2 V^T, 3 U on the rows of an Ml x ncols right-hand side share (M >= (Ml / v) Px v; Nl is not read), every column; op 4 W = U^T X V on
 * an Ml x Nl matrix share (covered; ncols is not read).  u / v: the r values of cflx_rbt_multipliers (depth x M each; the
 * side an op does not use may be NULL), formed into the library's s = fl(r fl(1/sqrt 2)) here.  ld >= ncols (op 4: Nl). */
int cflx_dbg_rbt_share(int op, const cflx_share_layout* share, int depth, const double* u, const double* v, int ncols,
                       double* share_inout, int ld);
/* cflx_chol_validate's per-share kernels on one layer-0 share A (tiled, non-empty; M = the larger of (Ml / v) Px v and
 * (Nl / v) Py v; Kappa >= 1); each output may be NULL:
 *   sumsq_out: the sum of squares of the entries with global row >= global column and global row < Kappa v;
 *   PT_out (v x ldp, ldp = Ml rounded up to even, + 2): the transposed panel of step t (0 <= t < Kappa, (t / Py + 1) v
 *   <= Nl) as the validation extracts it on grid column t % Py, PT[c][r] = A[row0 + r][(t / Py) v + c] (row0: the first
 *   local row of a tile with a global index >= t) where the global row is >= t v + c, else 0; its leading dimension is
 *   that of the broadcast piece (the active rows rounded up to even, >= 2).  Entries the kernel does not write, and all
 *   of PT off that grid column, are NaN. */
int cflx_dbg_chol_validate_share(const cflx_share_layout* share, const double* A, int t, double* PT_out, double* sumsq_out);
/* the two extract kernels of step t of cflx_lu_validate's sweep on one layer-0 share C of the packed factors (tiled,
 * non-empty, the LU's share of a square matrix: (Ml / v) Px == (Nl / v) Py, M = (Ml / v) Px v, Kappa = M / v; 0 <= t <
 * Kappa), under the sweep's owner guards; each output may be NULL, and entries the kernels do not write are NaN:
 *   LT_out (v x ldp, ldp = Ml rounded up to even; grid column t % Py): LT[c][r] = the unit lower factor's entry at the
 *   global row of r and global column t v + c, for the local rows r of tiles with a global index >= t;
 *   U_out (v x Nl; grid row t % Px): U[r][lc] = the upper factor's entry at global row t v + r and the global column of
 *   lc, for the local columns lc of tiles with a global index >= t. */
int cflx_dbg_lu_validate_share(const cflx_share_layout* share, const double* C, int t, double* LT_out, double* U_out);
/* the column-operand gather of the Cholesky trailing update on one share (tiled, non-empty; M and Kappa unused; pi is
 * not read but must lie on the grid like every position) at grid column pj, from the Px broadcast pieces of the
 * transposed panel of the global tiles >= gfirst: pieces holds piece p as v x ldp_p row-major, back to back, ldp_p =
 * the rows of grid row p's share from its first tile >= gfirst on, rounded up to even, >= 2 (what the factorisation
 * broadcasts). Bc_out (v x Nl): column tile t = the panel's rows of the global tile of the share's local column tile
 * lj0 + t, lj0 its first with a global index >= gfirst; NaN in the tiles after the last one. */
int cflx_dbg_chol_gather_cols(const cflx_share_layout* share, int gfirst, const double* pieces, double* Bc_out);
/* the assembly of the refinement's residual from the partials of the Px x Py x Pz ranks: all holds Px Py Pz chunks in
 * rank order ((pi Py + pj) Pz + pk), each ((nn ? Ml : 0) + (tn ? Nl : 0)) rows of 2 ldn (P then Q, or Hi then Lo; NN rows
 * first), of which only the layer-0 chunks are read; B, and each output (may be NULL), M x ldn.  Row g (tile T) adds the
 * NN partials of ranks (T % Px, pj, 0), pj ascending, then the TN partials of ranks (pi, T % Py, 0), pi ascending.
 * mode 0 (cflx_*_refine): R = b - p, ratio and W as LAPACK dgerfs; 1 (cflx_*_refine_x): R, ratio as dla_lin_berr and
 * Q = q; 2 (cflx_*_refine_x): R = b - (the double-double sum of the (Hi, Lo) pairs), rounded once.  Entries outside the
 * first nrhs columns, and outputs a mode does not write, are NaN. */
int cflx_dbg_refine_assemble(int mode, int Px, int Py, int Pz, int v, int M, int Ml, int Nl, int nn, int tn, int nrhs,
                             int ldn, const double* all, const double* B, double* R_out, double* ratio_out, double* W_out,
                             double* Q_out);
/* the refinement's per-column steps on M x ldn row-major host arrays A and D (first nrhs columns), sel: ldn ints; each
 * output may be NULL:
 *   max_out (nrhs): the maximum of each column of A, NaN wins;
 *   stats_out (nrhs x 5): {max |y|, max |y| d, max |dy| d, max |dy| / |y| (+inf where y = 0 != dy), min |y|} of y = A,
 *   dy = D (d: M scales, NULL: ones), NaN wins;
 *   select_out: A where sel[c] != 0, else 0;  add_out: A + D where sel[c] != 0, else A;
 *   Y_out, T_inout (both or neither): (A, T) updated by D with how = sel: 1 y += dy, 2 (y, t) += dy as LAPACK
 *   dla_wwaddw, 0 unchanged. */
int cflx_dbg_refine_columns(int M, int ldn, int nrhs, const double* A, const double* D, const double* d, const int* sel,
                            double* max_out, double* stats_out, double* select_out, double* add_out, double* Y_out,
                            double* T_inout);
/* the product kernel of cflx_lu_det / cflx_chol_det on host vectors of n doubles: d, and the divisors s1, s2 (may be
 * NULL).  mant_out 2^exp_out = |prod d| (square = 1: its square) divided by |prod s1| and |prod s2| (squared too), in the
 * kernel's fixed order; neg_out: the parity of the negative entries of d, s1 and s2 (0 when square); first_zero_out: 1 +
 * the first index with d_i == 0, or 0; nonfinite_out: 1 when an entry of d that is inf or NaN, or of a divisor that is
 * inf, NaN or zero, comes before the first zero (mant is then NaN; with a zero and no such entry before it, mant is 0).
 * Any output may be NULL. */
int cflx_dbg_det(int n, const double* d, const double* s1, const double* s2, int square, double* mant_out,
                 int64_t* exp_out, int* neg_out, int* first_zero_out, int* nonfinite_out);
/* partial-pivot LU of an n x v row-major panel: perm_out[v], A00_out[v*v] (L00\U00), LU_out[n*v] rows unpermuted */
int cflx_dbg_panel(int n, int v, const double* panel, int* perm_out, double* A00_out, double* LU_out, int reps,
                   double* ms_out);
/* X = B * U^-1 (right, upper, non-unit; B n x v) and Y = L^-1 * R (left, lower, unit; R v x n), A00 = L\U packed.
 * nb: the diagonal block size (4, 8, ..., 128 dividing v; 0 = the factorisation's default choice).  ld: the leading
 * dimension of the K-major panels on the device (even, >= n rounded up to even; 0 = that minimum); their padding
 * columns hold NaN. */
int cflx_dbg_trsm(int n, int v, int nb, int64_t ld, const double* A00, const double* B, double* X_out, const double* R,
                  double* Y_out);
/* inverses of the nb x nb diagonal blocks of A00 = L\U (v x v, nb in 4, 8, ..., 128, v % nb == 0) as the TRSMs use them:
 * Uinv_out[v / nb][nb][nb] = inv(U_jj), LinvT_out[v / nb][nb][nb] = inv(L_jj)^T (L unit lower); only the blocks are read */
int cflx_dbg_diag_inverse(int v, int nb, const double* A00, double* Uinv_out, double* LinvT_out);
/* Cholesky of one v x v row-major tile (lower triangle read) as the factorisation runs it.  variant 0: one-CTA kernel,
 * 4 <= v <= 512; 1: the 128 x 128 block kernel, v == 128; 2: the 128-block tile driver, v % 128 == 0 and v >= 256.
 * L_out = L with zeros above the diagonal, LT_out = L^T, info_out = 1 + first non-positive pivot's column, or 0. */
int cflx_dbg_potrf_tile(int v, const double* A, double* L_out, double* LT_out, int* info_out, int variant);
/* Unpivoted LU of one v x v row-major block as cflx_lu_factor_fixed runs it (4 <= v <= 1024, v % 4 == 0).  variant 0:
 * the one-CTA kernel on the whole block; 1: the 128-block driver (v % 128 == 0, v >= 256, what the factorisation runs
 * there: 128 x 128 diagonal blocks on the one-CTA kernel, the rest on the TRSMs and the FP64 GEMM).  LU_out = L\U with unit L, pivots |u| < tiny replaced by copysign(tiny, u) (+tiny for
 * +-0), nrepl_out (may be NULL) = the replacements, info_out = 1 + the first exactly zero pivot's column, or 0. */
int cflx_dbg_getrf_nopiv_tile(int v, const double* A, double tiny, double* LU_out, int* nrepl_out, int* info_out,
                              int variant);
/* D = C - AT^T * B on the int8 wgmma path (error-free digit planes, ozaki.cu); K % 128 == 0, N even.  AT is
 * [K x (row0 + M)] and B [K x (col0 + N)]: the planes of every row / column are made, the product takes operand rows
 * [row0, row0 + M) and columns [col0, col0 + N), on at most max_ctas CTAs (0 = one per SM).  C/D [M x N].  Optional test
 * outputs: digit planes [8][row0 + M][K] / [8][col0 + N][K], exponents [row0 + M] / [col0 + N].  ms_out / split_ms_out:
 * mean device time of the GEMM kernel / of the digit-plane kernels. */
int cflx_dbg_ozaki_gemm(int M, int N, int K, int row0, int col0, int max_ctas, const double* AT, const double* B,
                        const double* C, double* D, signed char* planesA_out, signed char* planesB_out, int* ea_out,
                        int* eb_out, int reps, double* ms_out, double* split_ms_out);
/* raw int8 tensor-core rate of back-to-back wgmma (64 x n x 32, n = 64/128/192/256, operands resident in shared memory,
 * two warpgroups per CTA, one CTA per SM).  tmacs_out = tera-MACs/s (x2 = TOP/s). */
int cflx_dbg_wgmma_peak(int n, double* tmacs_out);
/* plan_moves + push_phase1..3 + gri bookkeeping on one rank: the npiv pivot rows (local indices >= fnpr, tournament
 * order) are pushed to rows [fnpr, fnpr+npiv) exactly like push_pivots_up (conflux_opt.hpp:176-218, tests/unit/
 * test_utils.cpp:8-84).  n_cols even.  gri_out[n_rows] = new row -> old row, a01_out[npiv*n_cols] = extracted rows. */
int cflx_dbg_push_pivots(int n_rows, int n_cols, double* A_inout, int npiv, const int* pivot_rows, int fnpr, int* gri_out,
                         double* a01_out);
/* raw FP64 pipe micro-benchmarks, TFLOP/s: which = 0 the MMA shape gemm_tn_kernel issues (mma.sync m16n8k8 f64),
 * 1 DFMA, 2 / 3 / 4 mma.sync m16n8k4 / m16n8k8 / m16n8k16 f64, 5 mma.sync m8n8k4 f64 */
int cflx_dbg_fp64_peak(int which, double* tflops_out);
/* same probe: burst (best of ~2 ms launches) and sustained (one ~0.5 s launch, power-capped) TFLOP/s */
int cflx_dbg_fp64_peak_ex(int which, double* burst_out, double* sustained_out);

#ifdef __cplusplus
}
#endif
#endif /* CONFLUX_B200_H */
