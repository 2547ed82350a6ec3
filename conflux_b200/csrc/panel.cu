// conflux_b200/csrc/panel.cu -- tournament-pivot panel factorisation kernel (K1 of SURVEY.md 2.3).
//
// Replaces LUP = LAPACKE_dgetrf(ROW_MAJOR, n, v) + ipiv->perm at
// /root/reference/src/conflux/lu/conflux_opt.hpp:143-166 (called at :727 for the local candidates and at :291 for
// every 2v x v tournament round).  Only two things of that factorisation are kept by the reference: the winners
// perm[0..v) and (last round) the top v x v block L00\U00; this kernel produces exactly those.
//
// Design (GPU-first, not a LAPACK translation):
//   * the panel is stored TRANSPOSED, W[c][r]: a pivot search over column c is a coalesced scan of one row of W;
//   * one persistent cooperative grid (<= 132 CTAs, one per SM of an H100); owner thread <-> matrix row; rows NEVER move: LAPACK's
//     interchanges are tracked as a per-row "position" so that idamax tie-breaking (first maximal |a| in the
//     swapped order) is reproduced exactly (needed for the reference's integer test matrices);
//   * right-looking with an NB-column inner block held in shared memory; per column ONE grid-wide exchange:
//     every CTA publishes its best candidate together with that row's inner-block values into a double-buffered
//     global slot as "LL" words (payload + epoch in one 8-byte volatile store: the flag travels with the data), then
//     polls all headers, picks the winner redundantly and reads the winner's row from its slot -- two dependent L2
//     round trips per column, no reply from the owner, no grid barrier.
//     A CTA is 8 row-owner warps plus one GATHER WARP that owns no rows.  On grids of <= 32 CTAs (every look-ahead launch)
//     the gather warp alone runs the exchange of column j+1 -- one slot per lane, warp argmax, row fetch, 1 / pivot --
//     from the moment the candidate is published, while the owners apply the rest of elimination j; the block barrier
//     that publishes the winner's row is the one rendezvous of the column.  Slot reuse: column j+2 reuses the slot
//     parity of column j.  A CTA publishes j+2 only after its rendezvous of column j+1, which its gather warp reaches
//     only once EVERY CTA has published j+1, and a CTA publishes j+1 only after its own rendezvous of column j, i.e.
//     after its gather warp has consumed every word of column j it reads.  So no word of column j is overwritten
//     while a reader still needs it (model: oracle/panel_exchange_ref.py).  Larger grids poll with all threads and reduce with a block argmax.
//     The LL words order only their own payload; the trailing columns of W that phase C writes with plain stores and
//     that OTHER CTAs gather as pivot rows one block later are ordered by a gpu-scope fence pair per NB-column block
//     (writer: __threadfence() after the phase-C write-back; reader: __threadfence() before the U12 gathers);
//   * warp-level argmax with redux.sync on the (hi, lo) words of |a| and the position;
//   * after NB columns each CTA redundantly solves U12 = L11^-1 A12 (NB x rem, shared memory) and applies the
//     rank-NB update to its own rows with the multipliers in registers; CTA 0 emits the rows of L00\U00.
#include <cooperative_groups.h>

#include <climits>
#include <cstdlib>

#include "common.cuh"
#include "kernels.h"

namespace cflx {

namespace {
constexpr int PT_THREADS = 256;  // 8 row-owner warps: two per scheduler, so dependent DFMA/LDS chains of one warp are covered
constexpr int PT_WARPS = PT_THREADS / 32;
constexpr int PT_LAUNCH = PT_THREADS + 32;  // + the gather warp, which owns no rows (warp PT_WARPS)
constexpr int PT_ALLWARPS = PT_LAUNCH / 32;
constexpr int MAXG = 132;   // SMs of an H100 SXM
constexpr int RPT_LIMIT = 8;  // rows per thread -> R <= 1024 rows per CTA

struct PanelArgs {
    double* W;
    int64_t ldw;
    int n, v, nsteps;
    int R, Rpad, G;
    int* perm_out;
    double* A00;  // may be null: rows of L00\U00 from the pivot's inner block on
    uint2* slot_hdr;   // [2][MAXG][4]  LL words {payload32, epoch}: val_lo, val_hi, pos, row
    uint2* slot_rows;  // [2][MAXG][64] LL words: inner-block row of the candidate, two words per double
    int epoch_base;
};

// "LL" exchange (flag travels with the data in one 8-byte word, so no fence / separate flag / L1 invalidate):
__device__ __forceinline__ void st_ll(uint2* p, unsigned data, unsigned epoch) {
    asm volatile("st.volatile.global.v2.u32 [%0], {%1, %2};" ::"l"(p), "r"(data), "r"(epoch) : "memory");
}
__device__ __forceinline__ uint4 ld_ll2(const uint2* p) {  // two consecutive LL words
    uint4 v;
    asm volatile("ld.volatile.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
    return v;
}

struct Cand {
    unsigned long long key;  // bits of |a| (monotone for non-negative doubles)
    int pos;                 // LAPACK position (tie-break: smaller wins); INT_MAX = no candidate
    int row;
};

__device__ __forceinline__ Cand warp_argmax(Cand c) {
    const unsigned hi = (unsigned)(c.key >> 32), lo = (unsigned)c.key;
    const unsigned m1 = __reduce_max_sync(0xffffffffu, hi);
    bool in = (hi == m1);
    const unsigned m2 = __reduce_max_sync(0xffffffffu, in ? lo : 0u);
    in = in && (lo == m2);
    const unsigned m3 = __reduce_min_sync(0xffffffffu, in ? (unsigned)c.pos : (unsigned)INT_MAX);
    const unsigned ballot = __ballot_sync(0xffffffffu, in && (unsigned)c.pos == m3);
    const int src = __ffs(ballot) - 1;
    Cand r;
    r.key = ((unsigned long long)m1 << 32) | m2;
    r.pos = (int)m3;
    r.row = __shfl_sync(0xffffffffu, c.row, src);
    return r;
}
__device__ __forceinline__ bool better(const Cand& a, const Cand& b) {  // a strictly better than b
    return a.key > b.key || (a.key == b.key && a.pos < b.pos);
}
// block-wide argmax over all PT_ALLWARPS warps; result identical in every thread.  red_* have 2 x PT_ALLWARPS entries and
// `rb` alternates between the two halves on every call, so ONE barrier per reduction is enough (the buffer of call i is
// rewritten by call i+2, which every thread reaches only after the barrier of call i+1).  The per-warp results are
// reduced by a second warp_argmax (one entry per lane) in every warp: three shared loads and the redux chain instead
// of 3 x PT_ALLWARPS dependent loads and compares per thread.
__device__ __forceinline__ Cand block_argmax(Cand c, unsigned long long* red_key, int* red_pos, int* red_row, int& rb) {
    Cand w = warp_argmax(c);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int o = rb * PT_ALLWARPS;
    rb ^= 1;
    if (lane == 0) {
        red_key[o + warp] = w.key;
        red_pos[o + warp] = w.pos;
        red_row[o + warp] = w.row;
    }
    __syncthreads();
    Cand x{0ull, INT_MAX, -1};
    if (lane < PT_ALLWARPS) x = Cand{red_key[o + lane], red_pos[o + lane], red_row[o + lane]};
    return warp_argmax(x);
}

template <int NB, int RPT_MAX>
__global__ void __launch_bounds__(PT_LAUNCH, 1) panel_getrf_kernel(PanelArgs p) {
    // layout and size: panel_smem_bytes<NB>
    extern __shared__ __align__(16) unsigned char smem_raw[];
    double* Ab = reinterpret_cast<double*>(smem_raw);  // [NB][Rpad] inner block, column-major per CTA
    double* U12 = Ab + (size_t)NB * p.Rpad;            // [NB][v]
    double* LU11 = U12 + (size_t)NB * p.v;             // [NB][NB+1] LU rows of this block's pivots
    double* prow = LU11 + NB * (NB + 1);               // [2][NB + 1] winner row and 1 / pivot, double-buffered by column parity
    unsigned long long* red_key = reinterpret_cast<unsigned long long*>(prow + 2 * (NB + 1));
    int* red_pos = reinterpret_cast<int*>(red_key + 2 * PT_ALLWARPS);
    int* red_row = red_pos + 2 * PT_ALLWARPS;
    int* pivrow_blk = red_row + 2 * PT_ALLWARPS;  // [NB]
    int* win_sh = pivrow_blk + NB;  // [2][2] winner {pos, row} broadcast by the gathering warp, by column parity
    unsigned char* s_act = reinterpret_cast<unsigned char*>(win_sh + 4);  // [Rpad] row still active?
    int rb = 0;

    const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
    // Threads 0..PT_THREADS-1 own rows.  The last warp owns none: on grids of <= 32 CTAs it alone runs the exchange (one
    // slot per lane), so the poll of column j+1 starts at once while the row owners still apply elimination j.  Larger
    // grids poll with every thread and reduce with a block argmax.
    const bool owner = t < PT_THREADS;
    const bool small = p.G <= 32;
    const bool fetcher = warp == (small ? PT_WARPS : 0);  // the warp that fetches the winner's row
    const int cta = blockIdx.x;
    const int row_base = cta * p.R;
    const int Rloc = max(0, min(p.R, p.n - row_base));
    const int Rpad = p.Rpad, v = p.v;
    double* __restrict__ W = p.W;
    const int64_t ldw = p.ldw;

    int pos[RPT_MAX];
    bool active[RPT_MAX];
#pragma unroll
    for (int q = 0; q < RPT_MAX; ++q) {
        const int lr = t + q * PT_THREADS;
        pos[q] = row_base + lr;
        active[q] = owner && lr < Rloc;
    }
    for (int lr = t; lr < Rpad; lr += PT_LAUNCH) s_act[lr] = lr < Rloc ? 1 : 0;

    for (int jb = 0; jb < p.nsteps; jb += NB) {
        const int nbc = min(NB, v - jb);         // columns in this block
        const int nsb = min(nbc, p.nsteps - jb);  // elimination steps in this block
        // ---- phase A: load the inner block of my rows (coalesced rows of W) ----
        for (int e = t; e < nbc * Rpad; e += PT_LAUNCH) {  // all threads, coalesced along the rows of W
            const int c = e / Rpad, lr = e - c * Rpad;
            if (lr < Rloc) Ab[e] = W[(int64_t)(jb + c) * ldw + row_base + lr];
        }
        __syncthreads();
        // (each thread touches only its own rows of Ab until a winner row is published after a block sync)

        // ---- phase B: nsb pivot steps, software-pipelined across columns ----
        // The candidate of column j+1 is found and PUBLISHED as soon as the multipliers of column j are known (only
        // column j+1 of the inner block is updated first); the row owners apply the remaining columns of elimination j
        // while the exchange is in flight, so its latency hides the rank-1 update instead of adding to it.
        auto local_candidate = [&](int col) -> Cand {
            Cand c{0ull, INT_MAX, -1};
#pragma unroll
            for (int q = 0; q < RPT_MAX; ++q) {
                const int lr = t + q * PT_THREADS;
                if (active[q]) {
                    Cand o{(unsigned long long)__double_as_longlong(fabs(Ab[col * Rpad + lr])), pos[q], row_base + lr};
                    if (better(o, c)) c = o;
                }
            }
            return block_argmax(c, red_key, red_pos, red_row, rb);
        };
        // publish my CTA's candidate for global column jg and its inner-block row (LL words, fire and forget).  jprev >= 0:
        // elimination jprev has been applied to column jprev+1 only; the other trailing columns of the candidate's row
        // are eliminated on the fly with the SAME fma the owner thread will apply later (pw = winner row of jprev).
        auto publish = [&](const Cand& mine, int jg, int jprev, const double* pw) {
            const unsigned epoch = (unsigned)(p.epoch_base + jg + 1);
            const int par = jg & 1;
            uint2* myhdr = p.slot_hdr + (size_t)(par * MAXG + cta) * 4;
            if (t < 4) {
                const unsigned w = t == 0 ? (unsigned)mine.key : t == 1 ? (unsigned)(mine.key >> 32)
                                 : t == 2 ? (unsigned)mine.pos : (unsigned)mine.row;
                st_ll(myhdr + t, w, epoch);
            }
            if (t < nbc) {  // (zeros when this CTA has no active row left: only the winner's row words are read)
                double x = 0.0;
                if (mine.row >= 0) {
                    const int lrw = mine.row - row_base;
                    x = Ab[t * Rpad + lrw];
                    if (jprev >= 0 && t > jprev + 1) x = fma(-Ab[jprev * Rpad + lrw], pw[t], x);
                }
                const unsigned long long xb = (unsigned long long)__double_as_longlong(x);
                uint2* myrow = p.slot_rows + (size_t)(par * MAXG + cta) * 64 + 2 * t;
                st_ll(myrow, (unsigned)xb, epoch);
                st_ll(myrow + 1, (unsigned)(xb >> 32), epoch);
            }
        };
        {
            const Cand mine0 = local_candidate(0);
            if (t < 32) __threadfence();  // publisher-side half of the per-block release of my phase-C stores (cumulative)
            publish(mine0, jb, -1, nullptr);
        }
        for (int j = 0; j < nsb; ++j) {
            const int jg = jb + j;
            const int par = jg & 1;
            double* pr = prow + par * (NB + 1);  // the winner's inner-block row, then 1 / pivot
            if (!small || fetcher) {
                // gather every CTA's candidate for column jg, pick the winner, fetch its inner-block row.  G <= 32: the
                // gather warp alone (one slot per lane, warp-level argmax, no block barrier); larger grids poll with all warps.
                const unsigned epoch = (unsigned)(p.epoch_base + jg + 1);
                Cand gc{0ull, INT_MAX, -1};
                for (int g = small ? lane : t; g < p.G; g += small ? 32 : PT_LAUNCH) {
                    const uint2* h = p.slot_hdr + (size_t)(par * MAXG + g) * 4;
                    uint4 a, b;
                    do {
                        a = ld_ll2(h);
                        b = ld_ll2(h + 2);
                    } while (a.y != epoch || a.w != epoch || b.y != epoch || b.w != epoch);
                    Cand o{((unsigned long long)a.z << 32) | a.x, (int)b.x, (int)b.z};
                    if (better(o, gc)) gc = o;
                }
                const Cand w = small ? warp_argmax(gc) : block_argmax(gc, red_key, red_pos, red_row, rb);
                // (w.row < 0 cannot happen while jg < nsteps = min(n, v): some row is still active)
                // the winner's slot: on the gather warp (one slot per lane) the lane that held its row, no integer division
                const int wslot = small ? __ffs(__ballot_sync(0xffffffffu, gc.row == w.row)) - 1 : w.row / p.R;
                if (fetcher && lane < nbc) {  // the winner's row: second L2 round trip
                    const uint2* wr = p.slot_rows + (size_t)(par * MAXG + wslot) * 64 + 2 * lane;
                    uint4 a;
                    do {
                        a = ld_ll2(wr);
                    } while (a.y != epoch || a.w != epoch);
                    const double x = __longlong_as_double((long long)(((unsigned long long)a.z << 32) | a.x));
                    // safe before the barrier below: prow and win_sh are double-buffered by column parity, and the last
                    // reader of prow[par] (elimination jg - 2) finished before the barrier of column jg - 1, which this
                    // warp passed before it began this gather; LU11 row j is read only by phase C and the A00 emission,
                    // after the block's later barriers
                    pr[lane] = x;
                    LU11[j * (NB + 1) + lane] = x;
                    if (lane == j) pr[NB] = x != 0.0 ? 1.0 / x : 0.0;  // one IEEE division per CTA instead of one per thread
                }
                if (fetcher && lane == 0) {
                    win_sh[2 * par] = w.pos;
                    win_sh[2 * par + 1] = w.row;
                }
            }
            __syncthreads();  // winner + its row are in shared memory; every thread has finished elimination j-1
            Cand win;
            win.key = 0;
            win.pos = win_sh[2 * par];
            win.row = win_sh[2 * par + 1];
            if (t == 0) {
                pivrow_blk[j] = win.row;
                if (cta == 0) p.perm_out[jg] = win.row;
            }
            const double pivot = pr[j];
            const double rinv = pr[NB];
            const bool have_next = (j + 1 < nbc);
            const double pnext = have_next ? pr[j + 1] : 0.0;
            double lq[RPT_MAX];
#pragma unroll
            for (int q = 0; q < RPT_MAX; ++q) {
                const int lr = t + q * PT_THREADS;
                lq[q] = 0.0;
                if (!active[q]) continue;
                if (row_base + lr == win.row) {
                    active[q] = false;
                    s_act[lr] = 0;
                    continue;
                }
                if (pos[q] == jg) pos[q] = win.pos;  // the row that sat at position jg moves to the winner's slot
                if (pivot != 0.0) {
                    lq[q] = Ab[j * Rpad + lr] * rinv;
                    Ab[j * Rpad + lr] = lq[q];
                }
                if (have_next) Ab[(j + 1) * Rpad + lr] = fma(-lq[q], pnext, Ab[(j + 1) * Rpad + lr]);  // next column first
            }
            if (j + 1 < nsb) {
                const Cand mine = local_candidate(j + 1);  // (its block barrier also orders the multiplier stores above)
                publish(mine, jg + 1, j, pr);
                __syncthreads();  // the candidate row's pre-update values have been read before its owner updates them
            }
            if (owner) {
                double* __restrict__ ab = Ab;
#pragma unroll 4
                for (int c2 = j + 2; c2 < nbc; ++c2) {
                    const double pc = pr[c2];
#pragma unroll
                    for (int q = 0; q < RPT_MAX; ++q) {
                        const int lr = t + q * PT_THREADS;
                        if (active[q]) ab[c2 * Rpad + lr] = fma(-lq[q], pc, ab[c2 * Rpad + lr]);
                    }
                }
            }
        }

        // ---- write the inner block back (L multipliers; pivot rows keep their LU row) ----
        __syncthreads();  // every row's inner block is final
        for (int e = t; e < nbc * Rpad; e += PT_LAUNCH) {
            const int c = e / Rpad, lr = e - c * Rpad;
            if (lr < Rloc) W[(int64_t)(jb + c) * ldw + row_base + lr] = Ab[e];
        }
        if (cta == 0 && p.A00 != nullptr) {
            for (int e = t; e < nsb * nbc; e += PT_LAUNCH) {
                const int i = e / nbc, c = e % nbc;
                p.A00[(size_t)(jb + i) * v + jb + c] = LU11[i * (NB + 1) + c];
            }
        }

        // ---- phase C: U12 = L11^-1 A12, trailing columns of my rows -= L21 * U12 ----
        const int cstart = jb + nbc;
        const int rem = v - cstart;
        if (rem > 0) {
            __syncthreads();  // pivrow_blk, LU11 complete
            __threadfence();  // acquire: the epochs observed in phase B order the owners' earlier W stores before my gathers
            // one trailing column per thread: NB independent scattered loads in flight, then the unit-lower forward
            // substitution entirely in registers (L11 broadcast from shared memory)
            for (int cc = t; cc < rem; cc += PT_LAUNCH) {
                const double* col = W + (int64_t)(cstart + cc) * ldw;
                double u[NB];
#pragma unroll
                for (int i = 0; i < NB; ++i) u[i] = (i < nsb) ? ld_cg_f64(col + pivrow_blk[i]) : 0.0;
#pragma unroll
                for (int i = 1; i < NB; ++i) {
                    if (i < nsb) {
#pragma unroll
                        for (int s2 = 0; s2 < i; ++s2) u[i] -= LU11[i * (NB + 1) + s2] * u[s2];
                    }
                }
#pragma unroll
                for (int i = 0; i < NB; ++i) U12[i * v + cc] = u[i];
                if (cta == 0 && p.A00 != nullptr) {
#pragma unroll
                    for (int i = 0; i < NB; ++i)
                        if (i < nsb) p.A00[(size_t)(jb + i) * v + cstart + cc] = u[i];
                }
            }
            __syncthreads();
            // rank-NB update of my rows.  One thread per (row, column group): with R >= 256 rows per CTA a thread walks
            // all trailing columns of its row(s); with fewer rows the PT_THREADS / R threads that share a row split the
            // columns (groups of 4, interleaved), so small panels still use every thread of every CTA.
            auto update_row = [&](int lr, int cfirst, int cstep, bool tail) {
                double l[NB];
#pragma unroll
                for (int i = 0; i < NB; ++i) l[i] = (i < nsb) ? Ab[i * Rpad + lr] : 0.0;
                double* wp = W + (int64_t)cstart * ldw + row_base + lr;
                int cc = cfirst;
                // software-pipelined: the loads of the next group are issued before the FMAs of the current one
                double w0 = 0, w1 = 0, w2 = 0, w3 = 0;
                if (cc + 3 < rem) {
                    w0 = wp[(int64_t)cc * ldw];
                    w1 = wp[(int64_t)(cc + 1) * ldw];
                    w2 = wp[(int64_t)(cc + 2) * ldw];
                    w3 = wp[(int64_t)(cc + 3) * ldw];
                }
                for (; cc + 3 < rem; cc += cstep) {
                    double n0 = 0, n1 = 0, n2 = 0, n3 = 0;
                    const int cn = cc + cstep;
                    if (cn + 3 < rem) {
                        n0 = wp[(int64_t)cn * ldw];
                        n1 = wp[(int64_t)(cn + 1) * ldw];
                        n2 = wp[(int64_t)(cn + 2) * ldw];
                        n3 = wp[(int64_t)(cn + 3) * ldw];
                    }
#pragma unroll
                    for (int i = 0; i < NB; ++i) {
                        const double2 ua = *reinterpret_cast<const double2*>(U12 + i * v + cc);
                        const double2 ub = *reinterpret_cast<const double2*>(U12 + i * v + cc + 2);
                        w0 -= l[i] * ua.x;
                        w1 -= l[i] * ua.y;
                        w2 -= l[i] * ub.x;
                        w3 -= l[i] * ub.y;
                    }
                    wp[(int64_t)cc * ldw] = w0;
                    wp[(int64_t)(cc + 1) * ldw] = w1;
                    wp[(int64_t)(cc + 2) * ldw] = w2;
                    wp[(int64_t)(cc + 3) * ldw] = w3;
                    w0 = n0;
                    w1 = n1;
                    w2 = n2;
                    w3 = n3;
                }
                if (tail) {
                    for (int ct = rem & ~3; ct < rem; ++ct) {
                        double x = wp[(int64_t)ct * ldw];
#pragma unroll
                        for (int i = 0; i < NB; ++i) x -= l[i] * U12[i * v + ct];
                        wp[(int64_t)ct * ldw] = x;
                    }
                }
            };
            if (RPT_MAX == 1 && p.R < PT_THREADS) {
                const int nshare = PT_THREADS / p.R;  // threads per row
                const int lr = t % p.R, part = t / p.R;
                if (owner && part < nshare && lr < Rloc && s_act[lr]) update_row(lr, 4 * part, 4 * nshare, part == 0);
            } else {
#pragma unroll 1
                for (int q = 0; q < RPT_MAX; ++q) {
                    const int lr = t + q * PT_THREADS;
                    if (lr >= Rloc || !active[q]) continue;  // finished pivot rows are never read again
                    update_row(lr, 0, 4, true);
                }
            }
        }
        // release: my phase-C stores to W must be visible gpu-wide before any LL word of the NEXT block is published
        // (other CTAs gather these rows as pivot rows after observing that block's epochs)
        __threadfence();
        __syncthreads();  // Ab / U12 / LU11 are rewritten by the next block
    }
    // identity tail of perm (n < v): LAPACK leaves perm[i] = i for i >= n (conflux_opt.hpp:150-165)
    if (cta == 0)
        for (int i = p.nsteps + t; i < v; i += PT_LAUNCH) p.perm_out[i] = i;
}

// =====================================================================================================================
// Small panels (n <= 1024 rows: the 2v x v stacks of the tournament rounds, conflux_opt.hpp:291, and the last local
// panels): COLUMN-block owners instead of row owners.  A 1024-row column block of 16 columns fits the registers of one
// CTA (one row per thread), so the pivot search over such a block needs NO exchange between CTAs at all: two block
// barriers per column instead of an L2 round trip.  CTA c owns columns [16c, 16c+16): it applies the published blocks
// b < c to its columns (right-looking, U12 by forward substitution with the publisher's L11, then the rank-16 update from
// registers), factors its own block, writes it back in place and raises flag c.  The chain that matters is
// publish(b) -> update + factor in CTA b+1 -> publish(b+1); every other CTA trails behind it.  Logical CTA ids are handed
// out by an atomic ticket, so a CTA only ever waits for CTAs that started before it (no co-residency requirement).
// Arithmetic = the same fma chain per element, in the same order, as panel_getrf_kernel: results are bit-identical.
constexpr int SK_CB = 16;
struct StackArgs {
    double* W;
    int64_t ldw;
    int n, v;
    int* perm_out;      // [v]
    int* ppos;          // [v] LAPACK position of pivot j at the time it was chosen (replays the interchanges)
    unsigned* flags;    // [v / SK_CB] == epoch once the block is published
    unsigned* ticket;
    unsigned ticket_base, epoch;
};
__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_u32(unsigned* p, unsigned v) {
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void cp_async16(double* smem_dst, const double* gsrc) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

template <int NT>
__global__ void __launch_bounds__(NT, 1) stack_getrf_kernel(StackArgs p) {
    __shared__ double A12s[SK_CB][SK_CB + 1];  // pivot rows of block b in my columns, then U12
    __shared__ double L11s[SK_CB][SK_CB + 1];  // their multipliers inside block b
    __shared__ double prow[2][SK_CB];
    __shared__ unsigned long long red_key[2][32];
    __shared__ int red_pos[2][32], red_row[2][32];
    __shared__ int pivs[SK_CB], ppos_s[SK_CB];
    __shared__ int s_cta;
    extern __shared__ __align__(16) double Ls[];  // [SK_CB][NT] multipliers of the block being applied, row t in column t
    const int t = threadIdx.x, warp = t >> 5, lane = t & 31, nw = blockDim.x >> 5;
    if (t == 0) s_cta = (int)(atomicAdd(p.ticket, 1u) - p.ticket_base);
    __syncthreads();
    const int c = s_cta, c0 = c * SK_CB;
    const bool valid = t < p.n;
    double* __restrict__ W = p.W;
    const int64_t ldw = p.ldw;
    double a[SK_CB];
#pragma unroll
    for (int j = 0; j < SK_CB; ++j) a[j] = valid ? W[(int64_t)(c0 + j) * ldw + t] : 0.0;
    int pos = t;     // LAPACK position of my row (rows never move)
    int mypiv = -1;  // global pivot index once my row has been chosen

    for (int b = 0; b < c; ++b) {
        if (t == 0)
            while (ld_acquire_u32(p.flags + b) != p.epoch) {}
        __syncthreads();  // block b is published (and nobody still reads the shared tiles of the previous block)
        if (t < SK_CB) {
            pivs[t] = ld_cg_s32(p.perm_out + b * SK_CB + t);
            ppos_s[t] = ld_cg_s32(p.ppos + b * SK_CB + t);
        }
        // the multipliers of block b (n x 16) go straight into shared memory with 16-byte asynchronous copies (.cg: L2 only --
        // a stale L1 line must never serve data another CTA published); no registers are held while the round trip is in
        // flight and it overlaps the forward substitution below.  Thread (h, q) copies rows 2q, 2q+1 of columns 8h..8h+7.
        {
            const int half = blockDim.x >> 1, q = t % half, h = t / half;
            if (2 * q < p.n) {
                const double* lp = W + (int64_t)(b * SK_CB + 8 * h) * ldw + 2 * q;
#pragma unroll
                for (int k = 0; k < SK_CB / 2; ++k) cp_async16(Ls + (8 * h + k) * NT + 2 * q, lp + (int64_t)k * ldw);
            }
        }
        cp_async_commit();
        __syncthreads();
        int kk = -1;
        if (mypiv < 0) {
#pragma unroll
            for (int k = 0; k < SK_CB; ++k) {
                if (pivs[k] == t) kk = k;
                else if (kk < 0 && pos == b * SK_CB + k) pos = ppos_s[k];  // my row is swapped into the winner's old place
            }
        }
        if (kk >= 0) {
#pragma unroll
            for (int j = 0; j < SK_CB; ++j) A12s[kk][j] = a[j];
#pragma unroll
            for (int k = 0; k < SK_CB; ++k) L11s[kk][k] = ld_cg_f64(W + (int64_t)(b * SK_CB + k) * ldw + t);
        }
        __syncthreads();
        if (t < SK_CB) {  // U12 = L11^-1 A12 in place, one column per thread, the same fma chain as phase C of panel_getrf_kernel
#pragma unroll
            for (int i = 1; i < SK_CB; ++i) {
                double x = A12s[i][t];
#pragma unroll
                for (int s2 = 0; s2 < i; ++s2) x = fma(-L11s[i][s2], A12s[s2][t], x);
                A12s[i][t] = x;
            }
        }
        cp_async_wait_all();
        __syncthreads();
        if (kk >= 0) {  // my row is pivot kk of block b: it keeps its U values
#pragma unroll
            for (int j = 0; j < SK_CB; ++j) a[j] = A12s[kk][j];
            mypiv = b * SK_CB + kk;
        } else if (mypiv < 0 && valid) {
#pragma unroll
            for (int k = 0; k < SK_CB; ++k) {
                const double lk = Ls[k * NT + t];
#pragma unroll
                for (int j = 0; j < SK_CB; ++j) a[j] = fma(-lk, A12s[k][j], a[j]);
            }
        }
    }

    // ---- my own block: partial pivoting entirely inside the CTA ----
#pragma unroll
    for (int j = 0; j < SK_CB; ++j) {
        const int jg = c0 + j, par = j & 1;
        Cand cd{0ull, INT_MAX, -1};
        if (valid && mypiv < 0) cd = Cand{(unsigned long long)__double_as_longlong(fabs(a[j])), pos, t};
        const Cand w1 = warp_argmax(cd);
        if (lane == 0) {
            red_key[par][warp] = w1.key;
            red_pos[par][warp] = w1.pos;
            red_row[par][warp] = w1.row;
        }
        __syncthreads();
        Cand x{0ull, INT_MAX, -1};
        if (lane < nw) x = Cand{red_key[par][lane], red_pos[par][lane], red_row[par][lane]};
        const Cand win = warp_argmax(x);  // identical in every warp
        if (t == win.row) {
#pragma unroll
            for (int m = 0; m < SK_CB; ++m) prow[par][m] = a[m];
            mypiv = jg;
        }
        if (t == 0) {
            p.perm_out[jg] = win.row;
            p.ppos[jg] = win.pos;
        }
        __syncthreads();
        if (valid && mypiv < 0) {
            if (pos == jg) pos = win.pos;
            const double pivot = prow[par][j];
            const double rinv = pivot != 0.0 ? 1.0 / pivot : 0.0;
            double lq = 0.0;
            if (pivot != 0.0) {
                lq = a[j] * rinv;
                a[j] = lq;
            }
#pragma unroll
            for (int m = j + 1; m < SK_CB; ++m) a[m] = fma(-lq, prow[par][m], a[m]);
        }
    }
    if (valid) {
#pragma unroll
        for (int j = 0; j < SK_CB; ++j) W[(int64_t)(c0 + j) * ldw + t] = a[j];
    }
    __threadfence();
    __syncthreads();
    if (t == 0) st_release_u32(p.flags + c, p.epoch);
}

int launch_stack_getrf(double* W, int64_t ldw, int n, int v, int* perm_out, PanelWorkspace* ws, cudaStream_t stream) {
    StackArgs a{};
    a.W = W;
    a.ldw = ldw;
    a.n = n;
    a.v = v;
    a.perm_out = perm_out;
    a.ppos = ws->sk_ppos;
    a.flags = ws->sk_flags;
    a.ticket = ws->sk_ticket;
    a.ticket_base = ws->sk_ticket_count;
    a.epoch = ++ws->sk_epoch;
    const int C = v / SK_CB;
    ws->sk_ticket_count += (unsigned)C;
    const int threads = (int)round_up(n, 32);
    static PerDeviceMax cfg;
    if (cfg.raise((size_t)SK_CB * 1024 * sizeof(double))) {
        CFLX_CUDA(cudaFuncSetAttribute(stack_getrf_kernel<1024>, cudaFuncAttributeMaxDynamicSharedMemorySize, SK_CB * 1024 * 8));
        CFLX_CUDA(cudaFuncSetAttribute(stack_getrf_kernel<512>, cudaFuncAttributeMaxDynamicSharedMemorySize, SK_CB * 512 * 8));
    }
    if (threads <= 256) stack_getrf_kernel<256><<<C, threads, SK_CB * 256 * sizeof(double), stream>>>(a);
    else if (threads <= 512) stack_getrf_kernel<512><<<C, threads, SK_CB * 512 * sizeof(double), stream>>>(a);
    else stack_getrf_kernel<1024><<<C, threads, SK_CB * 1024 * sizeof(double), stream>>>(a);
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}

// the dynamic shared memory of panel_getrf_kernel<NB, *>, laid out in that order
template <int NB>
size_t panel_smem_bytes(int Rpad, int v) {
    return ((size_t)NB * Rpad + (size_t)NB * v + NB * (NB + 1) + 2 * (NB + 1)) * sizeof(double) +  // Ab, U12, LU11, prow
           2 * PT_ALLWARPS * (sizeof(unsigned long long) + 2 * sizeof(int)) +                     // red_key, red_pos, red_row
           (NB + 4) * sizeof(int) + (size_t)Rpad;                                           // pivrow_blk, win_sh, s_act
}

// Inner block size NB of the row-owner kernel: the first of 32, 16, 8, 4 that is <= v (4 always is) and satisfies
// (8 NB + 1) Rpad + 8 NB v <= 222 KiB - (8 NB^2 + 796 NB + 848).  These are the thresholds the kernel was validated and
// benchmarked with: they come from an earlier, larger shared-memory layout, so NB is smaller than panel_smem_bytes would
// allow for some shapes.  NB sets the blocking of the U12 solve and of the rank-NB update, and with it the rounding of
// the factors; raising it where it now fits is a change of its own that has to be measured.  0 = no NB fits.
int panel_nb(int Rpad, int v) {
    for (int nb = 32; nb >= 4; nb /= 2) {
        const long long limit = 222 * 1024 - (8LL * nb * nb + 796LL * nb + 848);
        if ((nb <= v || nb == 4) && (8LL * nb + 1) * Rpad + 8LL * nb * v <= limit) return nb;
    }
    return 0;
}

template <int NB, int RPT>
int launch_nb_rpt(PanelArgs& a, cudaStream_t stream) {
    const size_t smem = panel_smem_bytes<NB>(a.Rpad, a.v);
    void* params[] = {&a};
    static PerDeviceMax cfg;
    if (cfg.raise(smem))
        CFLX_CUDA(cudaFuncSetAttribute(panel_getrf_kernel<NB, RPT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    CFLX_CUDA(cudaLaunchCooperativeKernel((void*)panel_getrf_kernel<NB, RPT>, dim3(a.G), dim3(PT_LAUNCH), params, smem, stream));
    return CFLX_OK;
}
template <int NB>
int launch_nb(PanelArgs& a, cudaStream_t stream) {
    const int rpt = (a.R + PT_THREADS - 1) / PT_THREADS;
    if (rpt <= 1) return launch_nb_rpt<NB, 1>(a, stream);
    if (rpt <= 2) return launch_nb_rpt<NB, 2>(a, stream);
    if (rpt <= 4) return launch_nb_rpt<NB, 4>(a, stream);
    return launch_nb_rpt<NB, 8>(a, stream);
}
}  // namespace


int panel_workspace_create(PanelWorkspace* ws) {
    int dev = 0, sms = 0;
    CFLX_CUDA(cudaGetDevice(&dev));
    CFLX_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    ws->max_ctas = sms < MAXG ? sms : MAXG;
    ws->epoch = 1;
    ws->cta_cap = 0;
    CFLX_TRY(ws->slot_hdr.alloc_exact(2 * MAXG * 4));
    CFLX_TRY(ws->slot_rows.alloc_exact(2 * MAXG * 64));
    CFLX_CUDA(cudaMemset(ws->slot_hdr, 0, sizeof(uint2) * 2 * MAXG * 4));
    CFLX_CUDA(cudaMemset(ws->slot_rows, 0, sizeof(uint2) * 2 * MAXG * 64));
    // column-owner kernel for panels of <= 1024 rows: per-block flags, pivot positions, the CTA ticket
    CFLX_TRY(ws->sk_flags.alloc_exact(1024));
    CFLX_TRY(ws->sk_ppos.alloc_exact(16384));
    CFLX_TRY(ws->sk_ticket.alloc_exact(1));
    CFLX_CUDA(cudaMemset(ws->sk_flags, 0, sizeof(unsigned) * 1024));
    CFLX_CUDA(cudaMemset(ws->sk_ticket, 0, sizeof(unsigned)));
    ws->sk_epoch = 0;
    ws->sk_ticket_count = 0;
    {
        const char* e = getenv("CFLX_STACK_KERNEL");  // 0 = keep the row-owner kernel for small panels too
        ws->sk_enabled = e ? atoi(e) : 1;
    }
    return CFLX_OK;
}

// A00 (optional, v x v row-major) receives, for pivot i, the columns >= (i / NB) * NB of its L\U row; the
// caller completes the L prefix with launch_gather_a00 (which also needs perm).
int launch_panel_getrf_a00(double* W, int64_t ldw, int n, int v, int* perm_out, double* A00, int* nb_used,
                           PanelWorkspace* ws, cudaStream_t stream) {
    if (v <= 0 || n < 0) return CFLX_ERR_ARG;
    if (ws->sk_enabled && n >= v && n <= 1024 && v % SK_CB == 0 && v <= 16384 && ldw % 2 == 0 &&
        (reinterpret_cast<uintptr_t>(W) & 15) == 0) {
        if (nb_used) *nb_used = 0;  // nothing emitted into A00: launch_gather_a00 takes every entry from W
        return launch_stack_getrf(W, ldw, n, v, perm_out, ws, stream);
    }
    PanelArgs a{};
    a.W = W;
    a.ldw = ldw;
    a.n = n;
    a.v = v;
    a.nsteps = n < v ? n : v;
    // as many CTAs as the cap allows down to 32 rows per CTA: small panels (late steps, tournament stacks) are spread
    // over up to 32 SMs and the threads that share a row split the trailing columns in phase C
    int G = (n + 31) / 32;
    if (G < 1) G = 1;
    if (G > ws->max_ctas) G = ws->max_ctas;
    if (ws->cta_cap > 0 && G > ws->cta_cap) {
        G = ws->cta_cap;
        // the look-ahead cap must not shrink the row capacity below the panel: widen the grid again when needed
        const int need = (n + RPT_LIMIT * PT_THREADS - 1) / (RPT_LIMIT * PT_THREADS);
        if (G < need) G = need < ws->max_ctas ? need : ws->max_ctas;
    }
    int R = (n + G - 1) / G;
    R = (int)round_up(R > 0 ? R : 1, 32);
    G = n > 0 ? (n + R - 1) / R : 1;
    if (R > RPT_LIMIT * PT_THREADS) {
        set_last_error("panel_getrf: n=%d rows exceed the %d-row capacity (%d CTAs x %d rows)", n,
                       ws->max_ctas * RPT_LIMIT * PT_THREADS, ws->max_ctas, RPT_LIMIT * PT_THREADS);
        return CFLX_ERR_UNSUPPORTED;
    }
    a.R = R;
    a.Rpad = R;
    a.G = G;
    a.perm_out = perm_out;
    a.A00 = A00;
    a.slot_hdr = ws->slot_hdr;
    a.slot_rows = ws->slot_rows;
    a.epoch_base = ws->epoch;
    ws->epoch += v + 2 + (v & 1);  // keep the base even so slot parity == column parity
    const int nb = panel_nb(a.Rpad, v);
    if (nb == 0) {
        set_last_error("panel_getrf: v=%d with %d rows per CTA exceeds the shared-memory budget of the inner block", v,
                       a.Rpad);
        return CFLX_ERR_UNSUPPORTED;
    }
    if (nb_used) *nb_used = nb;
    switch (nb) {
        case 32: return launch_nb<32>(a, stream);
        case 16: return launch_nb<16>(a, stream);
        case 8: return launch_nb<8>(a, stream);
        default: return launch_nb<4>(a, stream);
    }
}

int launch_panel_getrf(double* W, int64_t ldw, int n, int v, int* perm_out, PanelWorkspace* ws, cudaStream_t stream) {
    return launch_panel_getrf_a00(W, ldw, n, v, perm_out, nullptr, nullptr, ws, stream);
}

}  // namespace cflx
