// examples/conflux_miniapp.cpp -- the reference's LU miniapp on the H100 path: same flags, same `_result_` line
// (reference: examples/conflux_miniapp.cpp:39-167).  Ranks are host threads of this process, one GPU each (the image
// has no MPI); a multi-process launcher would create the cflx_comm from an id shipped by its own transport instead.
//
//   conflux_miniapp -N 16384 -b 256 -r 2 [-p 2,2,1] [-t weak] [--validate]
// --validate (or building with -DCONFLUX_WITH_VALIDATION, the reference's compile-time switch) runs the reference's
// check after the last repetition -- P*A - L*U over the grid, "Total Frobenius norm" (conflux_miniapp.cpp:349-500) --
// on the GPUs and also prints the norm relative to ||A||_F.
#include <conflux/lu/conflux_b200.hpp>

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <iostream>
#include <thread>

int main(int argc, char** argv) {
    int N = 1000, b = 256, n_rep = 2, grid[3] = {-1, -1, -1};
    std::string type = "other";
#ifdef CONFLUX_WITH_VALIDATION
    bool validate = true;
#else
    bool validate = false;
#endif
    for (int i = 1; i < argc; ++i) {
        auto is = [&](const char* s, const char* l) { return !std::strcmp(argv[i], s) || !std::strcmp(argv[i], l); };
        if (is("-N", "--cols") && i + 1 < argc) N = std::atoi(argv[++i]);
        else if (is("-b", "--block_size") && i + 1 < argc) b = std::atoi(argv[++i]);
        else if (is("-r", "--n_rep") && i + 1 < argc) n_rep = std::atoi(argv[++i]);
        else if (is("-t", "--type") && i + 1 < argc) type = argv[++i];
        else if (is("-p", "--p_grid") && i + 1 < argc) std::sscanf(argv[++i], "%d,%d,%d", &grid[0], &grid[1], &grid[2]);
        else if (is("-l", "--print_limit") && i + 1 < argc) ++i;
        else if (is("--validate", "--validate")) validate = true;
        else if (is("-h", "--help")) {
            std::puts("conflux miniapp (H100): -N <cols> -b <block> -p Px,Py,Pz -r <reps> -t weak|strong|other");
            return 0;
        }
    }
    int ndev = 0;
    cflx_device_count(&ndev);
    int P = grid[0] > 0 ? grid[0] * grid[1] * grid[2] : (ndev > 0 ? 1 : 0);
    if (const char* e = std::getenv("CONFLUX_RANKS")) P = std::atoi(e);
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
            conflux::check(cflx_comm_create(P, r, P > 1 ? id : nullptr, r, &comm), "comm");
            {
                conflux::lu_params<double> params = grid[0] > 0
                    ? conflux::lu_params<double>(N, N, b, grid[0], grid[1], grid[2], comm)
                    : conflux::lu_params<double>(N, N, b, comm);
                if (params.rank == 0) {
                    std::cout << "======== INTERNAL PARAMS ========\nRank: 0, M: " << params.M << ", N: " << params.N
                              << ", P:" << params.P << ", v:" << params.v << ", Px:" << params.Px << ", Py: " << params.Py
                              << ", Pz: " << params.Pz << ", Nt: " << params.Nt << ", tA11x: " << params.tA11x
                              << ", tA11y: " << params.tA11y << "\n\n======== RESULT FORMAT ========\n"
                              << "_result_ lu,conflux,<num_rows>,<num_cols>,<num_ranks>,<process_grid>,time,other,<time_in_ms>,<block_size>\n\n"
                              << "======== RESULTS ========" << std::endl;
                }
                std::vector<int> piv(params.M);
                const int sqrtP = (int)std::sqrt((double)params.P);
                const int N_base = type == "weak" ? params.N / sqrtP : params.N;
                for (int i = 0; i < n_rep + 1; ++i) {  // i == 0 is the warm-up (conflux_miniapp.cpp:138-149)
                    params.InitMatrix();
                    std::size_t time = conflux::LU_rep<double>(params, nullptr, piv.data());
                    if (i > 0 && params.rank == 0)
                        std::cout << "_result_ lu,conflux," << params.N << "," << N_base << "," << params.P << "," << params.Px
                                  << "x" << params.Py << "x" << params.Pz << ",time," << type << "," << time << "," << params.v
                                  << std::endl;
                }
                if (validate) {  // collective; every rank gets the same numbers
                    double rel = 0;
                    const double frob = conflux::validate(params, &rel);
                    if (params.rank == 0) {
                        std::printf("Total Frobenius norm = %.4f\n", frob);
                        std::printf("Relative residual ||PA-LU||_F/||A||_F = %.3e\n", rel);
                        std::fflush(stdout);
                    }
                }
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
