// tests/cpp/layout_dump.hpp -- TEST INFRASTRUCTURE: one text format for a distributed-matrix descriptor, written both for
// the reference's costa::grid_layout (layout_dump_ref.cpp, golden data) and for this repo's conflux::grid_layout
// (layout_dump_mine.cpp, the test).  Local blocks are listed sorted by their global block coordinates (the order in which
// a layout enumerates them is an internal detail); `data` is printed as an element offset from the local buffer.
#pragma once
#include <algorithm>
#include <cstdio>
#include <string>
#include <tuple>
#include <vector>

struct DumpBlock {
    int row, col;
    long long offset;
    int stride, n_rows, n_cols;
};

inline std::string dump_layout(const std::string& key, const std::vector<int>& rows_split, const std::vector<int>& cols_split,
                               const std::vector<int>& owners, std::vector<DumpBlock> blocks) {
    std::string s = key + "\nrows";
    for (int x : rows_split) s += " " + std::to_string(x);
    s += "\ncols";
    for (int x : cols_split) s += " " + std::to_string(x);
    s += "\nowners";
    for (int x : owners) s += " " + std::to_string(x);
    s += "\n";
    std::sort(blocks.begin(), blocks.end(), [](const DumpBlock& a, const DumpBlock& b) { return std::tie(a.row, a.col) < std::tie(b.row, b.col); });
    char buf[160];
    for (const DumpBlock& b : blocks) {
        std::snprintf(buf, sizeof(buf), "block %d %d %lld %d %d %d\n", b.row, b.col, b.offset, b.stride, b.n_rows, b.n_cols);
        s += buf;
    }
    return s;
}
