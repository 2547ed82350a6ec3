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

}  // namespace conflux
