// conflux_b200/csrc/rbt.cu -- random butterfly transforms (cflx_lu_rbt, cflx_lu_rbt_solve, cflx_lu_rbt_apply_local):
// W = U^T A V with random recursive butterflies U and V of depth d (Parker 1995; Baboulin, Dongarra, Herrmann and Tomov,
// ACM TOMS 39(2), 2013; MAGMA's dgesv_rbt), so that W can be factored without the pivot search.
//
// Level l of a butterfly has blocks of n_l = M >> l rows and half h_l = n_l / 2; its matrix is diag over the blocks of
// (1/sqrt 2) [R0 R1; R0 -R1].  With s = fl(r fl(1/sqrt 2)) per row, the two operations on a row pair (p, q = p + h_l) are
//   transposed (B^T): x_p <- s_p (x_p + x_q),   x_q <- s_q (x_p - x_q)
//   forward    (B):   t_p = s_p x_p, t_q = s_q x_q;  x_p <- t_p + t_q,  x_q <- t_p - t_q
// each rounded once (__dmul_rn / __dadd_rn / __dsub_rn: nothing is contracted into an FMA, so the bits are numpy's).  U^T
// and V^T run the transposed operation at levels d-1 .. 0, U and V the forward one at levels 0 .. d-1; W runs, from level
// d-1 down to 0, the rows with U's level then the columns (the transposed operation along each row) with V's level.
//
// Locality: when 2^d v divides Ml (M a multiple of 2^d v Px), global rows i and i + (M >> (l+1)) are local rows r and
// r + (Ml >> (l+1)) of the same rank, and global block i / n_l is local block r / (Ml >> l); the same holds for the
// columns (Px == Py, Nl == Ml).  So every rank transforms its own share, with the multipliers of the global rows and
// columns it holds (Layout::row / col), and nothing is communicated.
//
// A thread takes the 2^n rows (2^n x 2^n entries for W) that n consecutive levels mix, and runs those levels on them in
// registers: depth 2 is one read and one write of the share, depth 3 and 4 two.
#include <climits>
#include <cmath>
#include <vector>

#include "lu_state.h"

namespace cflx {
namespace {

constexpr int RBT_THREADS = 128;
constexpr unsigned RBT_MAX_GRID_Y = 65535;

// the group of G = 2^NL indices that levels lo .. lo + NL - 1 mix, for group g of an n-long dimension: idx[k] =
// (g / hmin) (n >> lo) + g % hmin + k hmin, hmin = n >> (lo + NL) (the half of the finest level)
template <int NL>
__device__ __forceinline__ void group_of(int g, int n, int lo, int* idx) {
    const int hmin = n >> (lo + NL), base = (g / hmin) * (n >> lo) + g % hmin;
#pragma unroll
    for (int k = 0; k < (1 << NL); ++k) idx[k] = base + k * hmin;
}

// one level (the m-th of the group's NL) on one vector x of the group: pairs (k, k + st), st = 2^(NL-1-m);
// s: the multipliers of the group's indices at this level
template <int NL, bool FWD>
__device__ __forceinline__ void level_op(double* x, const double* s, int m) {
    const int st = 1 << (NL - 1 - m);
#pragma unroll
    for (int k = 0; k < (1 << NL); ++k) {
        if (k & st) continue;
        const double a = x[k], b = x[k + st];
        if (FWD) {
            const double ta = __dmul_rn(s[k], a), tb = __dmul_rn(s[k + st], b);
            x[k] = __dadd_rn(ta, tb);
            x[k + st] = __dsub_rn(ta, tb);
        } else {
            x[k] = __dmul_rn(s[k], __dadd_rn(a, b));
            x[k + st] = __dmul_rn(s[k + st], __dsub_rn(a, b));
        }
    }
}

// Rows only (RHS): levels lo .. lo + NL - 1 of one side on the rows of X (ld), a thread per (row group, local column c
// < ncols), columns with L.col(c) >= col_lim left alone; forward (ascending levels) or transposed (descending).
// Two-sided (W, !FWD): the same row groups crossed with the column groups of the Nl columns; at each level, U's rows
// (sr) then V's columns (sc).  sr / sc: d x M multipliers of the side, level l at l M.
template <int NL, bool FWD, bool TWO>
__global__ void __launch_bounds__(RBT_THREADS)
    rbt_kernel(double* __restrict__ X, int64_t ld, Layout L, int ncols, int col_lim, int lo,
               const double* __restrict__ sr, const double* __restrict__ sc) {
    constexpr int G = 1 << NL;
    const int nrg = L.Ml >> NL, ncg = TWO ? (ncols >> NL) : ncols;
    const int t = blockIdx.x * RBT_THREADS + threadIdx.x;
    if (t >= ncg) return;
    int cols[G];
    if (TWO) {
        group_of<NL>(t, ncols, lo, cols);
    } else {
        if (L.col(t) >= col_lim) return;
        cols[0] = t;
    }
    constexpr int NC = TWO ? G : 1;
    double scol[NL][G];
    if (TWO) {
#pragma unroll
        for (int m = 0; m < NL; ++m)
#pragma unroll
            for (int k = 0; k < G; ++k) scol[m][k] = sc[(int64_t)(lo + m) * L.M + L.col(cols[k])];
    }
    for (int g = blockIdx.y; g < nrg; g += gridDim.y) {
        int rows[G];
        group_of<NL>(g, L.Ml, lo, rows);
        double srow[NL][G];
#pragma unroll
        for (int m = 0; m < NL; ++m)
#pragma unroll
            for (int k = 0; k < G; ++k) srow[m][k] = sr[(int64_t)(lo + m) * L.M + L.row(rows[k])];
        double x[G][NC];  // x[row][col]
#pragma unroll
        for (int a = 0; a < G; ++a)
#pragma unroll
            for (int b = 0; b < NC; ++b) x[a][b] = X[(int64_t)rows[a] * ld + cols[b]];
#pragma unroll
        for (int i = 0; i < NL; ++i) {
            const int m = FWD ? i : NL - 1 - i;  // level lo + m
#pragma unroll
            for (int b = 0; b < NC; ++b) {
                double v[G];
#pragma unroll
                for (int a = 0; a < G; ++a) v[a] = x[a][b];
                level_op<NL, FWD>(v, srow[m], m);
#pragma unroll
                for (int a = 0; a < G; ++a) x[a][b] = v[a];
            }
            if (TWO) {
#pragma unroll
                for (int a = 0; a < G; ++a) level_op<NL, false>(x[a], scol[m], m);
            }
        }
#pragma unroll
        for (int a = 0; a < G; ++a)
#pragma unroll
            for (int b = 0; b < NC; ++b) X[(int64_t)rows[a] * ld + cols[b]] = x[a][b];
    }
}

template <int NL, bool FWD, bool TWO>
int launch_group(double* X, int64_t ld, const Layout& L, int ncols, int col_lim, int lo, const double* sr,
                 const double* sc, cudaStream_t s) {
    const int ncg = TWO ? (ncols >> NL) : ncols, nrg = L.Ml >> NL;
    if (ncg <= 0 || nrg <= 0) return CFLX_OK;
    const dim3 grid((ncg + RBT_THREADS - 1) / RBT_THREADS, std::min((unsigned)nrg, RBT_MAX_GRID_Y));
    rbt_kernel<NL, FWD, TWO><<<grid, RBT_THREADS, 0, s>>>(X, ld, L, ncols, col_lim, lo, sr, sc);
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}

template <bool FWD, bool TWO>
int launch_levels(double* X, int64_t ld, const Layout& L, int ncols, int col_lim, int depth, const double* sr,
                  const double* sc, cudaStream_t s) {
    // forward: levels (0, 1), (2, 3), ..; transposed: (d-1, d-2), (d-3, d-4), ..; a lone last level runs by itself
    for (int done = 0; done < depth;) {
        const int n = std::min(2, depth - done), lo = FWD ? done : depth - done - n;
        const int rc = n == 2 ? launch_group<2, FWD, TWO>(X, ld, L, ncols, col_lim, lo, sr, sc, s)
                              : launch_group<1, FWD, TWO>(X, ld, L, ncols, col_lim, lo, sr, sc, s);
        CFLX_TRY(rc);
        done += n;
    }
    return CFLX_OK;
}

// The mirror's tile moves (sym_mirror), one tile k of a list per blockIdx.y stride (the lists can be far longer than a
// grid's y extent); pack and transpose go through shared memory (transpose_tile):
//   pack:      buf[k][r][c] = A tile at (off[2k], off[2k + 1]) [c][r] (the tile transposed, contiguous)
//   unpack:    A tile at (off[2k], off[2k + 1]) [r][c] = buf[k][r][c]
//   transpose: A tile at (off[4k], off[4k + 1]) [r][c] = A tile at (off[4k + 2], off[4k + 3]) [c][r] (distinct tiles)
//   diag:      A tile at (off[2k], off[2k + 1]) [r][c] = the same tile [c][r] for c > r (upper from lower)
// D[r][c] = S[c][r] for one v x v tile, 32 x 32 blocks through shared memory (both sides coalesced): block blockIdx.x
// of the destination tile, a (32, 8) CTA
__device__ __forceinline__ void transpose_tile(const double* __restrict__ S, int64_t lds, double* __restrict__ D, int64_t ldd,
                                               int v, double (*t)[33]) {
    const int nbx = (v + 31) / 32, bi = blockIdx.x / nbx, bj = blockIdx.x % nbx;
    for (int y = threadIdx.y; y < 32; y += blockDim.y) {
        const int sr = bj * 32 + y, sc = bi * 32 + threadIdx.x;
        if (sr < v && sc < v) t[y][threadIdx.x] = S[(int64_t)sr * lds + sc];
    }
    __syncthreads();
    for (int y = threadIdx.y; y < 32; y += blockDim.y) {
        const int dr = bi * 32 + y, dc = bj * 32 + threadIdx.x;
        if (dr < v && dc < v) D[(int64_t)dr * ldd + dc] = t[threadIdx.x][y];
    }
    __syncthreads();
}
__global__ void tiles_pack_kernel(const double* __restrict__ A, int64_t ld, const int* __restrict__ off, int ntiles, int v,
                                  double* __restrict__ buf) {
    __shared__ double t[32][33];
    for (int k = blockIdx.y; k < ntiles; k += gridDim.y)
        transpose_tile(A + (int64_t)off[2 * k] * ld + off[2 * k + 1], ld, buf + (int64_t)k * v * v, v, v, t);
}
__global__ void tiles_unpack_kernel(const double* __restrict__ buf, const int* __restrict__ off, int ntiles, int v,
                                    double* __restrict__ A, int64_t ld) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= v * v) return;
    for (int k = blockIdx.y; k < ntiles; k += gridDim.y)
        A[(int64_t)(off[2 * k] + e / v) * ld + off[2 * k + 1] + e % v] = buf[(int64_t)k * v * v + e];
}
__global__ void tiles_transpose_kernel(double* __restrict__ A, int64_t ld, const int* __restrict__ off, int ntiles, int v) {
    __shared__ double t[32][33];
    for (int k = blockIdx.y; k < ntiles; k += gridDim.y)
        transpose_tile(A + (int64_t)off[4 * k + 2] * ld + off[4 * k + 3], ld, A + (int64_t)off[4 * k] * ld + off[4 * k + 1],
                       ld, v, t);
}
__global__ void tiles_diag_mirror_kernel(double* __restrict__ A, int64_t ld, const int* __restrict__ off, int ntiles, int v) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= v * v) return;
    const int r = e / v, c = e % v;
    if (c <= r) return;
    for (int k = blockIdx.y; k < ntiles; k += gridDim.y) {
        double* T = A + (int64_t)off[2 * k] * ld + off[2 * k + 1];
        T[(int64_t)r * ld + c] = T[(int64_t)c * ld + r];
    }
}
// the grid of a tile-list kernel: v^2 / 256 CTAs (transposes: one per 32 x 32 block) along x, the tiles along y
// (capped, the kernels stride)
dim3 tiles_grid(int v, size_t ntiles, bool transpose = false) {
    const unsigned x = transpose ? (unsigned)(((v + 31) / 32) * ((v + 31) / 32)) : (unsigned)((v * v + 255) / 256);
    return dim3(x, (unsigned)std::min<size_t>(ntiles, RBT_MAX_GRID_Y));
}

// splitmix64's finaliser (Steele, Lea and Flood, OOPSLA 2014)
uint64_t splitmix_final(uint64_t z) {
    z ^= z >> 30;
    z *= 0xBF58476D1CE4E5B9ull;
    z ^= z >> 27;
    z *= 0x94D049BB133111EBull;
    z ^= z >> 31;
    return z;
}
}  // namespace

void rbt_multipliers(int M, int depth, uint64_t seed, int side, double* r) {
    for (int l = 0; l < depth; ++l)
        for (int i = 0; i < M; ++i) {
            const uint64_t k = seed + 0x9E3779B97F4A7C15ull * ((((uint64_t)(2 * l + side)) << 32) + (uint64_t)i + 1);
            const double w = (double)(splitmix_final(k) >> 11) * 0x1p-53;
            r[(size_t)l * M + i] = std::exp((w - 0.5) / 10.0);
        }
}

void rbt_scales(const double* r, size_t n, double* s) {
    for (size_t i = 0; i < n; ++i) s[i] = r[i] * M_SQRT1_2;
}

int launch_rbt(RbtOp op, double* X, int64_t ld, const Layout& L, int ncols, int col_lim, int depth, const double* su,
               const double* sv, cudaStream_t s) {
    switch (op) {
        case RbtOp::UT: return launch_levels<false, false>(X, ld, L, ncols, col_lim, depth, su, nullptr, s);
        case RbtOp::V: return launch_levels<true, false>(X, ld, L, ncols, col_lim, depth, sv, nullptr, s);
        case RbtOp::VT: return launch_levels<false, false>(X, ld, L, ncols, col_lim, depth, sv, nullptr, s);
        case RbtOp::U: return launch_levels<true, false>(X, ld, L, ncols, col_lim, depth, su, nullptr, s);
        case RbtOp::W: return launch_levels<false, true>(X, ld, L, ncols, col_lim, depth, su, sv, s);
    }
    return refuse(__func__, "op is not an RbtOp");
}

int rbt_record_set(RbtRecord* dst, int depth, uint64_t seed, const double* s, int M, cudaStream_t st) {
    dst->depth = depth;
    dst->seed = seed;
    if (!depth) return CFLX_OK;
    const size_t n = 2 * (size_t)depth * M;
    CFLX_TRY(dst->s.grow(n));
    CFLX_CUDA(cudaMemcpyAsync(dst->s, s, sizeof(double) * n, cudaMemcpyDefault, st));
    return CFLX_OK;
}

int rbt_pass_on(RbtState* t, int M, bool next_is_plain, cudaStream_t s) {
    CFLX_TRY(rbt_record_set(&t->fac, t->in.depth, t->in.seed, t->in.s, M, s));
    if (next_is_plain) t->in.depth = 0;
    return CFLX_OK;
}

RowTransform rbt_rows(const Handle& h, RbtOp op) {
    const RbtRecord& f = h.rbt.fac;
    const Layout rows{h.M, h.v, h.Nt, h.M, 0, 1, 1, 0, 0};  // global row r is row r
    const double *su = f.s, *sv = f.s + (size_t)f.depth * h.M;
    cudaStream_t s = h.comm->stream;
    const int depth = f.depth;
    return [=](double* X, int64_t ld, int n) { return launch_rbt(op, X, ld, rows, n, INT_MAX, depth, su, sv, s); };
}

int rbt_apply_local(const char* who, const char* rbt_call, Handle* h, RbtOp op, int nrhs, double* B_local, int ldb) {
    CFLX_TRY(enter(h, who, NEED_FACTORS));
    const RbtRecord& f = h->rbt.fac;
    if (!f.depth) {
        set_last_error("%s: the factors carry no random butterfly transform (%s before the factorisation)", who, rbt_call);
        return CFLX_ERR_STATE;
    }
    const int ncl = rhs_local_cols(nrhs, h->v, h->Py);
    bool dev = false;
    CFLX_TRY(share_kind(who, *h, B_local, "B_local", &dev));
    cudaStream_t s = h->comm->stream;
    const size_t row = sizeof(double) * ncl;
    DevBuf<double> tmp;
    double* X = B_local;
    int64_t ld = ldb;
    if (!dev) {
        CFLX_TRY(tmp.alloc((size_t)h->Ml * ncl));
        CFLX_CUDA(cudaMemcpy2DAsync(tmp, row, B_local, sizeof(double) * ldb, row, h->Ml, cudaMemcpyHostToDevice, s));
        X = tmp;
        ld = ncl;
    }
    CFLX_TRY(launch_rbt(op, X, ld, *h, ncl, nrhs, f.depth, f.s, f.s + (size_t)f.depth * h->M, s));
    if (!dev) CFLX_CUDA(cudaMemcpy2DAsync(B_local, sizeof(double) * ldb, tmp, row, row, h->Ml, cudaMemcpyDeviceToHost, s));
    CFLX_CUDA(cudaStreamSynchronize(s));
    return CFLX_OK;
}

int sym_mirror(const Grid& g, double* A) {
    cflx_comm* c = g.comm;
    cudaStream_t s = c->stream;
    const int v = g.v, Px = g.Px, Py = g.Py, Nt = g.Nt, me = g.pi * Py + g.pj;
    const int npeer = Px * Py;
    // per other peer (grid position q = qi Py + qj of this layer), in the order (I, J) on both sides: the offsets of the
    // tiles (J, I) this rank sends and of the tiles (I, J) it receives; the pairs {(I, J), (J, I)} this rank holds both
    // of, transposed in place; the diagonal tiles it holds
    std::vector<std::vector<int>> snd(npeer), rcv(npeer);
    std::vector<int> loc, diag;
    for (int I = 0; I < Nt; ++I)
        for (int J = I; J < Nt; ++J) {
            const int dq = (I % Px) * Py + J % Py, sq = (J % Px) * Py + I % Py;
            if (I == J) {
                if (dq == me) diag.insert(diag.end(), {(I / Px) * v, (I / Py) * v});
            } else if (sq == me && dq == me) {
                loc.insert(loc.end(), {(I / Px) * v, (J / Py) * v, (J / Px) * v, (I / Py) * v});
            } else if (sq == me) {
                snd[dq].insert(snd[dq].end(), {(J / Px) * v, (I / Py) * v});
            } else if (dq == me) {
                rcv[sq].insert(rcv[sq].end(), {(I / Px) * v, (J / Py) * v});
            }
        }
    std::vector<int> off;  // the send list, the receive list (peers ascending), the local pairs, the diagonal tiles
    std::vector<size_t> sfirst(npeer + 1, 0), rfirst(npeer + 1, 0);
    for (int q = 0; q < npeer; ++q) {
        off.insert(off.end(), snd[q].begin(), snd[q].end());
        sfirst[q + 1] = sfirst[q] + snd[q].size() / 2;
    }
    for (int q = 0; q < npeer; ++q) {
        off.insert(off.end(), rcv[q].begin(), rcv[q].end());
        rfirst[q + 1] = rfirst[q] + rcv[q].size() / 2;
    }
    off.insert(off.end(), loc.begin(), loc.end());
    off.insert(off.end(), diag.begin(), diag.end());
    const size_t ns = sfirst[npeer], nr = rfirst[npeer], nl = loc.size() / 4, nd = diag.size() / 2, vv = (size_t)v * v;
    DevBuf<int> doff;
    CFLX_TRY(doff.alloc(off.size()));
    CFLX_CUDA(cudaMemcpyAsync(doff, off.data(), sizeof(int) * off.size(), cudaMemcpyHostToDevice, s));
    const int* d_loc = doff + 2 * (ns + nr);
    const int* d_diag = d_loc + 4 * nl;
    if (nl) tiles_transpose_kernel<<<tiles_grid(v, nl, true), dim3(32, 8), 0, s>>>(A, g.Nl, d_loc, (int)nl, v);
    CFLX_CUDA(cudaGetLastError());
    if (nd) tiles_diag_mirror_kernel<<<tiles_grid(v, nd), 256, 0, s>>>(A, g.Nl, d_diag, (int)nd, v);
    CFLX_CUDA(cudaGetLastError());
    if (ns + nr) {  // the tiles of other ranks: packed per peer, one group of sends and receives in this layer
        DevBuf<double> sbuf, rbuf;
        CFLX_TRY(sbuf.alloc(ns * vv));
        CFLX_TRY(rbuf.alloc(nr * vv));
        if (ns) tiles_pack_kernel<<<tiles_grid(v, ns, true), dim3(32, 8), 0, s>>>(A, g.Nl, doff, (int)ns, v, sbuf);
        CFLX_CUDA(cudaGetLastError());
        CFLX_NCCL(ncclGroupStart());
        for (int q = 0; q < npeer; ++q) {
            const int peer = q * g.Pz + g.pk;  // world rank of grid position q on this layer
            if (sfirst[q + 1] > sfirst[q])
                CFLX_NCCL(ncclSend(sbuf + sfirst[q] * vv, (sfirst[q + 1] - sfirst[q]) * vv, ncclDouble, peer, c->world, s));
            if (rfirst[q + 1] > rfirst[q])
                CFLX_NCCL(ncclRecv(rbuf + rfirst[q] * vv, (rfirst[q + 1] - rfirst[q]) * vv, ncclDouble, peer, c->world, s));
        }
        CFLX_NCCL(ncclGroupEnd());
        if (nr) tiles_unpack_kernel<<<tiles_grid(v, nr), 256, 0, s>>>(rbuf, doff + 2 * ns, (int)nr, v, A, g.Nl);
        CFLX_CUDA(cudaGetLastError());
        CFLX_CUDA(cudaStreamSynchronize(s));  // before the buffers are freed
    }
    CFLX_CUDA(cudaStreamSynchronize(s));  // the offsets are a temporary
    return CFLX_OK;
}

}  // namespace cflx

extern "C" int cflx_rbt_multipliers(int M, int depth, uint64_t seed, double* u_out, double* v_out) {
    REFUSE_IF(depth < 1);
    REFUSE_IF(depth > 4);
    REFUSE_IF(M < 1);
    REFUSE_IF(M % (1 << depth) != 0);
    REFUSE_IF(!u_out && !v_out);
    if (u_out) cflx::rbt_multipliers(M, depth, seed, 0, u_out);
    if (v_out) cflx::rbt_multipliers(M, depth, seed, 1, v_out);
    return CFLX_OK;
}
