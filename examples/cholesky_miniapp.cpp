// examples/cholesky_miniapp.cpp -- the reference's Cholesky miniapp on the H100 path: same flags, same report block
// (reference: examples/cholesky_miniapp.cpp:36-159).  Ranks are host threads of this process, one GPU each.
//
//   cholesky_miniapp --dim 32768 --tile 512 [--grid 4,2,1] [--run 5] [--ranks 8] [--validate]
// --ranks P (or the product of --grid) = number of GPUs; --validate prints ||A - L L^T||_F / ||A||_F after the last run.
#include <conflux/cholesky/conflux_b200_cholesky.hpp>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <iostream>
#include <thread>

static void printTimings(std::vector<double>& timings, std::ostream& out, int N, int v, conflux::ProcCoord grid[3]) {
    out << "==========================" << std::endl;
    out << "    PROBLEM PARAMETERS:" << std::endl;
    out << "==========================" << std::endl;
    out << "Matrix size: " << N << std::endl;
    out << "Tile size: " << v << std::endl;
    out << "Processor grid: " << grid[0] << "x" << grid[1] << "x" << grid[2] << std::endl;
    out << "Number of repetitions: " << timings.size() << std::endl;
    out << "--------------------------" << std::endl;
    out << "TIMINGS [ms] = ";
    for (auto& time : timings) out << time << " ";
    out << std::endl;
    out << "==========================" << std::endl;
}

int main(int argc, char** argv) {
    uint32_t N = 65536, v = 0, runs = 5;
    unsigned g[3] = {0, 0, 0};
    int P = -1;
    bool validate = false;
    for (int i = 1; i < argc; ++i) {
        auto is = [&](const char* s, const char* l) { return !std::strcmp(argv[i], s) || !std::strcmp(argv[i], l); };
        if (is("-N", "--dim") && i + 1 < argc) N = (uint32_t)std::atoi(argv[++i]);
        else if (is("-v", "--tile") && i + 1 < argc) v = (uint32_t)std::atoi(argv[++i]);
        else if (is("-r", "--run") && i + 1 < argc) runs = (uint32_t)std::atoi(argv[++i]);
        else if (is("-g", "--grid") && i + 1 < argc) std::sscanf(argv[++i], "%u,%u,%u", &g[0], &g[1], &g[2]);
        else if (is("--ranks", "--ranks") && i + 1 < argc) P = std::atoi(argv[++i]);
        else if (is("--validate", "--validate")) validate = true;
        else if (is("-h", "--help")) {
            std::puts("Cholesky Mini-App (H100): -N/--dim <n> -v/--tile <v> -g/--grid Px,Py,Pz -r/--run <runs> [--ranks P] [--validate]");
            return 0;
        }
    }
    int ndev = 0;
    cflx_device_count(&ndev);
    if (P < 0) P = g[0] ? (int)(g[0] * g[1] * g[2]) : (ndev > 0 ? 1 : 0);
    if (ndev < P || P < 1) {
        std::fprintf(stderr, "need %d CUDA devices, %d visible (no CPU fallback)\n", P, ndev);
        return 1;
    }
    unsigned char id[CFLX_UNIQUE_ID_BYTES] = {0};
    if (P > 1 && cflx_get_unique_id(id) != 0) {
        std::fprintf(stderr, "%s\n", cflx_last_error());
        return 1;
    }
    int status = 0;
    auto rank_main = [&](int r) {
        try {
            conflux::comm_t comm = nullptr;
            if (cflx_comm_create(P, r, P > 1 ? id : nullptr, r, &comm) != 0) throw conflux::CholeskyException(cflx_last_error());
            conflux::set_world(comm);
            conflux::ProcCoord grid[3] = {g[0], g[1], g[2]};
            // warm-up run (conflux cholesky_miniapp.cpp:104-108)
            conflux::initialize(argc, argv, N, v, grid);
            conflux::parallelCholesky();
            conflux::finalize(true);
            std::vector<double> timings;
            for (uint32_t i = 0; i < runs; ++i) {
                conflux::initialize(argc, argv, N, v, grid);
                conflux::parallelCholesky();
                timings.push_back((double)(long long)conflux::last_factorization_ms());
                if (validate && i + 1 == runs) {
                    double rel = 0;
                    conflux::validate(&rel);
                    if (conflux::world_rank() == 0) std::printf("Relative residual ||A-LL^T||_F/||A||_F = %.3e\n", rel);
                }
                const int nn = conflux::matrix_size(), vv = conflux::tile_size();
                const bool last = (i + 1 == runs);
                const int rk = conflux::world_rank();
                conflux::finalize(true);
                if (last && rk == 0) printTimings(timings, std::cout, nn, vv, grid);
            }
            cflx_comm_destroy(comm);
        } catch (const std::exception& e) {
            std::fprintf(stderr, "[rank %d] %s\n", r, e.what());
            status = 1;
        }
    };
    std::vector<std::thread> th;
    for (int r = 0; r < P; ++r) th.emplace_back(rank_main, r);
    for (auto& t : th) t.join();
    return status;
}
