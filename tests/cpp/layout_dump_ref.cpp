// tests/cpp/layout_dump_ref.cpp -- TEST INFRASTRUCTURE, used only by tests/golden/make_golden.py where the reference
// tree is present: prints the COSTA descriptors the REFERENCE's conflux_layout produces (src/conflux/lu/layout.cpp, both
// overloads; the 3-D one through lu_params::matrix on the thread-backed MPI stub) in the format of layout_dump.hpp.
#include <functional>
#include <random>

#include <conflux/lu/layout.hpp>
#include <conflux/lu/lu_params.hpp>

#include <cstdio>
#include <mutex>
#include <vector>

#include "layout_dump.hpp"

static std::string dump(costa::grid_layout<double>& g, const double* base, const std::string& key) {
    std::vector<int> rows, cols, owners;
    for (int i = 0; i < g.num_blocks_row(); ++i) rows.push_back(g.grid.rows_interval(i).start);
    rows.push_back(g.num_rows());
    for (int j = 0; j < g.num_blocks_col(); ++j) cols.push_back(g.grid.cols_interval(j).start);
    cols.push_back(g.num_cols());
    for (int i = 0; i < g.num_blocks_row(); ++i)
        for (int j = 0; j < g.num_blocks_col(); ++j) owners.push_back(g.grid.owner(i, j));
    std::vector<DumpBlock> blocks;
    for (size_t k = 0; k < g.blocks.num_blocks(); ++k) {
        auto& b = g.blocks.get_block(k);
        blocks.push_back({b.coordinates.row, b.coordinates.col, (long long)(b.data - base), b.stride, b.n_rows(), b.n_cols()});
    }
    return dump_layout(key, rows, cols, owners, blocks);
}

struct Case { int N, v, Px, Py, Pz; };
static std::mutex g_mu;
static std::vector<std::pair<int, std::string>> g_out;  // (cart rank, text): ranks are threads, printed in rank order

static void rank_main(int, void* p) {
    auto* c = (Case*)p;
    conflux::lu_params<double> params(c->N, c->N, c->v, c->Px, c->Py, c->Pz, MPI_COMM_WORLD);
    char key[160];
    std::snprintf(key, sizeof(key), "cart %d %d %d R %d %d %d %d %d %d", (int)params.M, (int)params.N, (int)params.v, (int)params.Px,
                  (int)params.Py, (int)params.Pz, (int)params.pi, (int)params.pj, (int)params.pk);
    std::string s = dump(params.matrix, params.data.data(), key);
    {
        std::lock_guard<std::mutex> lk(g_mu);
        g_out.push_back({(params.pi * params.Py + params.pj) * params.Pz + params.pk, s});
    }
    MPI_Barrier(params.lu_comm);
}

int main() {
    std::vector<double> buf(1 << 16);
    const int cases[][5] = {{16, 16, 4, 1, 1}, {64, 64, 8, 2, 2}, {96, 96, 8, 3, 3}, {48, 48, 4, 2, 2}};
    for (auto& c : cases)
        for (char ord : {'R', 'C'})
            for (int rank = 0; rank < c[3] * c[4]; ++rank) {
                auto ref = conflux::conflux_layout<double>(buf.data(), c[0], c[1], c[2], ord, c[3], c[4], rank);
                char key[160];
                std::snprintf(key, sizeof(key), "bc %d %d %d %c %d %d %d", c[0], c[1], c[2], ord, c[3], c[4], rank);
                std::fputs(dump(ref, buf.data(), key).c_str(), stdout);
            }
    Case cs[] = {{64, 8, 2, 2, 1}, {64, 8, 2, 2, 2}, {96, 8, 3, 3, 1}, {64, 16, 1, 1, 2}, {100, 16, 2, 2, 1}};
    for (auto& c : cs) {
        g_out.clear();
        stub_mpi_run(c.Px * c.Py * c.Pz, rank_main, &c);
        std::sort(g_out.begin(), g_out.end());
        for (auto& r : g_out) std::fputs(r.second.c_str(), stdout);
    }
    return 0;
}
