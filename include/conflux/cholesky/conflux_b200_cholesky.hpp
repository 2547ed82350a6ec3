// include/conflux/cholesky/conflux_b200_cholesky.hpp -- header-only C++ facade of the CONFCHOX path over the C ABI
// (include/conflux_b200.h, cflx_chol_*), keeping the reference's driver-facing names
//   conflux::initialize(argc, argv, N, v, grid) / conflux::parallelCholesky() / conflux::finalize(clean)
// (src/conflux/cholesky/Cholesky.h:20-22) so that examples/cholesky_miniapp.cpp reads like the reference's miniapp
// (examples/cholesky_miniapp.cpp:60-159 there).  The reference keeps its state in process globals (proc, prop, io,
// Cholesky.cpp:41-45) and talks to MPI_COMM_WORLD; here ranks may be threads of one process (one GPU each), so the state
// is thread-local and the world communicator is handed over once with conflux::set_world() (the MPI_Init analogue).
#pragma once
#include <cstdint>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../conflux_b200.h"

namespace conflux {

using ProcCoord = uint32_t;   // CholeskyTypes.h
using comm_t = cflx_comm*;

class CholeskyException : public std::runtime_error {
   public:
    explicit CholeskyException(const std::string& what) : std::runtime_error(what) {}
};

namespace chol_detail {
struct State {
    comm_t world = nullptr;
    cflx_chol* plan = nullptr;
    std::vector<double> data;   // this rank's share of the input (Ml x Nl, conflux tile layout)
    int info[16] = {0};
    double last_ms = 0;
};
inline State& state() {
    static thread_local State s;
    return s;
}
inline void check(int rc, const char* what) {
    if (rc != 0) throw CholeskyException(std::string(what) + ": " + cflx_last_error());
}
}  // namespace chol_detail

// replaces MPI_Init + MPI_COMM_WORLD: the communicator every later call of this thread refers to
inline void set_world(comm_t world) { chol_detail::state().world = world; }

// Cholesky.cpp:60-160.  grid = {0,0,0} and v = 0 are chosen for the user exactly like the reference does (and written
// back into grid); allocates the device buffers and generates the input (CholeskyIO.cpp:100-172).
inline void initialize(int /*argc*/, char* /*argv*/[], uint32_t N, uint32_t v, ProcCoord* grid) {
    auto& s = chol_detail::state();
    if (!s.world) throw CholeskyException("conflux::set_world() has not been called (the MPI_Init analogue)");
    if (s.plan) cflx_chol_destroy(s.plan);
    s.plan = nullptr;
    chol_detail::check(cflx_chol_create(s.world, (int)N, (int)v, (int)grid[0], (int)grid[1], (int)grid[2], &s.plan), "initialize");
    chol_detail::check(cflx_chol_info(s.plan, s.info), "initialize");
    grid[0] = (ProcCoord)s.info[7]; grid[1] = (ProcCoord)s.info[8]; grid[2] = (ProcCoord)s.info[9];
    s.data.assign((std::size_t)s.info[3] * s.info[4], 0.0);
    chol_detail::check(cflx_chol_init_matrix_host(s.info[0], s.info[1], s.info[7], s.info[8], s.info[9], s.info[13], s.data.data()),
                       "generateInputMatrixDistributed");
    chol_detail::check(cflx_chol_set_local(s.plan, s.data.data()), "initialize: upload");
}
// Cholesky.cpp:760-921: collective over the world communicator; the factor stays on the devices (cflx_chol_get_local)
inline void parallelCholesky() {
    auto& s = chol_detail::state();
    if (!s.plan) throw CholeskyException("parallelCholesky() before initialize()");
    chol_detail::check(cflx_chol_factor(s.plan, &s.last_ms), "parallelCholesky");
}
inline void finalize(bool clean = false) {
    auto& s = chol_detail::state();
    if (clean && s.plan) {
        cflx_chol_destroy(s.plan);
        s.plan = nullptr;
        s.data.clear();
        s.data.shrink_to_fit();
    }
}
// extras of the H100 path: device time of the last factorisation, tile size in use, grid-wide residual
inline double last_factorization_ms() { return chol_detail::state().last_ms; }
inline int tile_size() { return chol_detail::state().info[1]; }
inline int matrix_size() { return chol_detail::state().info[0]; }
inline int world_rank() { return chol_detail::state().info[13]; }
inline double validate(double* relative = nullptr) {
    double a = 0, r = 0;
    chol_detail::check(cflx_chol_validate(chol_detail::state().plan, &a, &r), "validate");
    if (relative) *relative = r;
    return a;
}
// A X = B with the factor of the last parallelCholesky() (cflx_chol_solve, collective; the reference has no solve).  B and
// X are matrix_size() x nrhs row-major; X may be nullptr on any rank.
inline void choleskySolve(int nrhs, const double* B, int ldb, double* X, int ldx) {
    auto& s = chol_detail::state();
    if (!s.plan) throw CholeskyException("choleskySolve() before initialize()");
    chol_detail::check(cflx_chol_solve(s.plan, nrhs, B, ldb, X, ldx), "choleskySolve");
}
// A X = B with the factor of the last parallelCholesky(), like ScaLAPACK's pdpotrs, with B and X distributed like A
// (cflx_chol_solve_local, collective): the shares and rules of conflux::LU_solve_local; only the rows of real tiles are
// read or written.
inline void choleskySolveLocal(int nrhs, const double* B_local, int ldb, double* X_local, int ldx) {
    auto& s = chol_detail::state();
    if (!s.plan) throw CholeskyException("choleskySolveLocal() before initialize()");
    chol_detail::check(cflx_chol_solve_local(s.plan, nrhs, B_local, ldb, X_local, ldx), "choleskySolveLocal");
}
// LAPACK dpocon of the last parallelCholesky() (cflx_chol_rcond, collective).  Returns the estimate of
// 1 / (||A||_1 ||A^-1||_1); *anorm = ||A||_1 of the padded symmetric input.
inline double choleskyRcond(double* anorm = nullptr) {
    auto& s = chol_detail::state();
    if (!s.plan) throw CholeskyException("choleskyRcond() before initialize()");
    double r = 0, a = 0;
    chol_detail::check(cflx_chol_rcond(s.plan, &r, &a), "choleskyRcond");
    if (anorm) *anorm = a;
    return r;
}
// LAPACK dporfs with the factor of the last parallelCholesky() (cflx_chol_refine, collective): X (matrix_size() x nrhs)
// holds a solution of A X = B and is refined in place; ferr / berr as conflux::LU_refine.
inline void choleskyRefine(int nrhs, const double* B, int ldb, double* X, int ldx, double* ferr = nullptr,
                           double* berr = nullptr) {
    auto& s = chol_detail::state();
    if (!s.plan) throw CholeskyException("choleskyRefine() before initialize()");
    chol_detail::check(cflx_chol_refine(s.plan, nrhs, B, ldb, X, ldx, ferr, berr), "choleskyRefine");
}
// LAPACK dporfsx with the factor of the last parallelCholesky() (cflx_chol_refine_x, collective): arguments and result
// as conflux::LU_refine_x without transposed.
inline int choleskyRefineX(int nrhs, const double* B, int ldb, double* X, int ldx, double* err_norm,
                           double* err_comp = nullptr, double* rcond = nullptr, double* berr = nullptr) {
    auto& s = chol_detail::state();
    if (!s.plan) throw CholeskyException("choleskyRefineX() before initialize()");
    int info = 0;
    chol_detail::check(cflx_chol_refine_x(s.plan, nrhs, B, ldb, X, ldx, rcond, berr, err_norm, err_comp, &info),
                       "choleskyRefineX");
    return info;
}
// LAPACK dpoequ (+ dlaqsy, lower, when apply) on the input the device holds (cflx_chol_equilibrate, collective); s
// (matrix_size()) may be null.  Returns info (0, or the first non-positive diagonal entry); equed is 'N' or 'Y'.
inline int choleskyEquilibrate(bool apply = true, double* s_out = nullptr, double* scond = nullptr, double* amax = nullptr,
                               char* equed = nullptr) {
    auto& s = chol_detail::state();
    if (!s.plan) throw CholeskyException("choleskyEquilibrate() before initialize()");
    int info = 0;
    chol_detail::check(cflx_chol_equilibrate(s.plan, apply ? 1 : 0, s_out, scond, amax, equed, &info), "choleskyEquilibrate");
    return info;
}
// LAPACK dposvx after parallelCholesky(), with the scaling the factor carries (cflx_chol_svx, collective); ferr / berr /
// equed may be null.  Returns info (0, or N + 1 when rcond < 2^-53).
inline int choleskySvx(int nrhs, const double* B, int ldb, double* X, int ldx, double* rcond, double* ferr = nullptr,
                       double* berr = nullptr, char* equed = nullptr) {
    auto& s = chol_detail::state();
    if (!s.plan) throw CholeskyException("choleskySvx() before initialize()");
    int info = 0;
    chol_detail::check(cflx_chol_svx(s.plan, nrhs, B, ldb, X, ldx, rcond, ferr, berr, equed, &info), "choleskySvx");
    return info;
}
// LAPACK dpoequb (+ dlaqsy, lower, when apply) on the input the device holds (cflx_chol_equilibrate_b, collective):
// choleskyEquilibrate with the scales rounded to powers of two.
inline int choleskyEquilibrateB(bool apply = true, double* s_out = nullptr, double* scond = nullptr,
                                double* amax = nullptr, char* equed = nullptr) {
    auto& s = chol_detail::state();
    if (!s.plan) throw CholeskyException("choleskyEquilibrateB() before initialize()");
    int info = 0;
    chol_detail::check(cflx_chol_equilibrate_b(s.plan, apply ? 1 : 0, s_out, scond, amax, equed, &info),
                       "choleskyEquilibrateB");
    return info;
}
// LAPACK dposvxx after parallelCholesky(), with the scaling the factor carries (cflx_chol_svxx, collective): arguments
// and result as conflux::LU_svxx without transposed.
inline int choleskySvxx(int nrhs, const double* B, int ldb, double* X, int ldx, double* rcond, double* err_norm,
                        double* err_comp = nullptr, double* rpvgrw = nullptr, double* berr = nullptr,
                        char* equed = nullptr) {
    auto& s = chol_detail::state();
    if (!s.plan) throw CholeskyException("choleskySvxx() before initialize()");
    int info = 0;
    chol_detail::check(cflx_chol_svxx(s.plan, nrhs, B, ldb, X, ldx, rcond, rpvgrw, berr, err_norm, err_comp, equed, &info),
                       "choleskySvxx");
    return info;
}
// LAPACK dpotri (lower) with the factor of the last parallelCholesky() (cflx_chol_inverse, collective): Ainv_local (Ml x
// Nl; host or device memory; may be null) receives inv(A) on this rank's real tiles on and below the diagonal, zeros
// elsewhere.
inline void choleskyInverse(double* Ainv_local) {
    auto& s = chol_detail::state();
    if (!s.plan) throw CholeskyException("choleskyInverse() before initialize()");
    chol_detail::check(cflx_chol_inverse(s.plan, Ainv_local), "choleskyInverse");
}
// log det(A) = 2 sum log l_ii of the last parallelCholesky() (cflx_chol_det, collective); det = *mant * 2^*exp.  unscaled:
// divided by prod(s)^2 of the scaling the factor carries (choleskyEquilibrate).  mant / exp may be null.
inline double choleskyLogdet(bool unscaled = false, double* mant = nullptr, int64_t* exp = nullptr) {
    auto& s = chol_detail::state();
    if (!s.plan) throw CholeskyException("choleskyLogdet() before initialize()");
    double ld = 0;
    chol_detail::check(cflx_chol_det(s.plan, unscaled ? 1 : 0, &ld, mant, exp), "choleskyLogdet");
    return ld;
}

}  // namespace conflux
