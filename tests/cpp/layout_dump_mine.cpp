// tests/cpp/layout_dump_mine.cpp -- TEST INFRASTRUCTURE: reads layout keys from stdin (the key lines of
// tests/golden/layout_ref.txt) and prints this repo's conflux_layout descriptor for each, in the format of layout_dump.hpp.
//   bc   M N v ordering Px Py rank           conflux_layout(data, M, N, v, ordering, Px, Py, rank)
//   cart M N v ordering Px Py Pz pi pj pk    conflux_layout(data, M, N, v, ordering, lu_comm) on the 3-D grid
#include <conflux/lu/conflux_b200.hpp>

#include <iostream>
#include <sstream>

#include "layout_dump.hpp"

static std::string dump(const conflux::grid_layout<double>& g, const double* base, const std::string& key) {
    std::vector<DumpBlock> blocks;
    for (const conflux::block_t& b : g.localblocks)
        blocks.push_back({b.row, b.col, (long long)(static_cast<const double*>(b.data) - base), b.ld,
                          g.rowsplit[b.row + 1] - g.rowsplit[b.row], g.colsplit[b.col + 1] - g.colsplit[b.col]});
    return dump_layout(key, g.rowsplit, g.colsplit, g.owners, blocks);
}

int main() {
    std::vector<double> buf(1 << 20);
    std::string line;
    while (std::getline(std::cin, line)) {
        std::istringstream in(line);
        std::string kind;
        int M, N, v, Px, Py;
        char ord;
        in >> kind >> M >> N >> v >> ord >> Px >> Py;
        if (kind == "bc") {
            int rank;
            in >> rank;
            std::cout << dump(conflux::conflux_layout<double>(buf.data(), M, N, v, ord, Px, Py, rank), buf.data(), line);
        } else if (kind == "cart") {
            conflux::cart_t c;
            c.dims[0] = Px; c.dims[1] = Py;
            in >> c.dims[2] >> c.coords[0] >> c.coords[1] >> c.coords[2];
            c.rank = c.cart_rank(c.coords[0], c.coords[1], c.coords[2]);
            std::cout << dump(conflux::conflux_layout<double>(buf.data(), M, N, v, ord, c), buf.data(), line);
        }
    }
    return 0;
}
