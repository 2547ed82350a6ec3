// conflux_b200/csrc/lu.cu -- host orchestration of the CONFLUX LU step loop on H100 + the C ABI.
//
// One rank = one GPU = one host thread/process (SPMD, like the reference's MPI ranks).  The step order follows
// conflux::LU_rep<T> (/root/reference/src/conflux/lu/conflux_opt.hpp:535-1803, blueprint in SURVEY.md appendix A)
// but the data layout and the division of labour are GPU-first:
//   * A11 stays resident in HBM (row-major Ml x Nl, 64-bit indexing); L and U are written IN PLACE into it
//     (the reference keeps a second Ml x Nl array A10resultBuff + a caller-owned C and MPI_Puts into it);
//   * panels are kept transposed/K-major (see gemm.cu, panel.cu) so every kernel streams contiguous rows;
//   * pivot rows are gathered by ONE sum-reduction over the (i,k) plane of zero-padded v x ncols buffers
//     (exact: every row has exactly one non-zero contributor per layer) instead of reduce + p2p gather
//     (conflux_opt.hpp:1164-1173,1226-1258,1474-1511); A00 and the pivot ids travel in one broadcast
//     (conflux_opt.hpp:818-850,872);
//   * all communication is NCCL on the rank's stream; at Px == 1 the whole factorisation is enqueued without a
//     single host synchronisation, at Px > 1 the host reads back one int (this rank's pivot count) per step.
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdarg>
#include <cstdlib>
#include <cstring>
#include <random>
#include <string>
#include <vector>

#include <nvtx3/nvToolsExt.h>

#include "lu_state.h"

namespace cflx {
static thread_local char g_err[1024] = "";
void set_last_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
}  // namespace cflx

using namespace cflx;

namespace {
int flipbit(int n, int k) { return n ^ (1 << k); }
int butterfly_pair(int pi, int r, int Px) {  // conflux_opt.cpp:59-72
    int src = flipbit(pi, r);
    if (src >= Px) {
        if (r == 0) src = pi;
        else {
            src = flipbit(src, r - 1);
            if (src >= Px) src = Px - 1;
        }
    }
    return src;
}
#include "init_tables.inc"
// decodes the fixed input matrix of size n x n (row-major) if the reference has one
bool fixed_input_matrix(int n, std::vector<double>* out) {
    for (const InitTable& t : kInitTables) {
        if (t.n != n) continue;
        out->clear();
        out->reserve((size_t)n * n);
        if (t.kind == 0) {
            for (const char* p = t.text; *p; ++p) out->push_back((double)(*p - '0'));
        } else {
            const char* p = t.text;
            while (*p) {
                char* e = nullptr;
                out->push_back(std::strtod(p, &e));
                p = (*e == ',') ? e + 1 : e;
            }
        }
        return out->size() == (size_t)n * n;
    }
    return false;
}
int pick_nb(int v) {  // block size of the diagonal inverses / TRSM sweeps (template instances: 128, 64, 32, 16, 8, 4)
    static int cap = -1;  // CFLX_TRSM_NB caps the block size (A/B switch; default 128)
    if (cap < 0) {
        const char* e = getenv("CFLX_TRSM_NB");
        cap = e ? atoi(e) : 128;
    }
    for (int nb : {128, 64, 32, 16, 8, 4})
        if (nb <= cap && v % nb == 0) return nb;
    return 0;
}
}  // namespace

namespace cflx {
int make_sub(cflx_comm* c, int color, int key, int size, SubComm* out) {
    out->size = size;
    out->rank = key;
    out->c = nullptr;
    if (c->world_size == 1) return CFLX_OK;
    // every rank takes part in every split (collective over the world communicator)
    CFLX_NCCL(ncclCommSplit(c->world, color, key, &out->c, nullptr));
    int r = -1, s = -1;
    CFLX_NCCL(ncclCommUserRank(out->c, &r));
    CFLX_NCCL(ncclCommCount(out->c, &s));
    if (r != key || s != size) {
        set_last_error("sub-communicator mismatch: rank %d/%d expected %d/%d", r, s, key, size);
        return CFLX_ERR_NCCL;
    }
    return CFLX_OK;
}
int grid_barrier(cflx_comm* c) {
    if (c->world_size > 1)
        CFLX_NCCL(ncclAllReduce(c->d_scratch, c->d_scratch, 1, ncclDouble, ncclSum, c->world, c->stream));
    CFLX_CUDA(cudaStreamSynchronize(c->stream));
    return CFLX_OK;
}
int grid_init(Grid* g, cflx_comm* c, int Px, int Py, int Pz) {
    g->comm = c;
    g->Px = Px; g->Py = Py; g->Pz = Pz; g->P = Px * Py * Pz;
    g->rank = c->world_rank;
    g->pi = g->rank / (Py * Pz);
    g->pj = (g->rank / Pz) % Py;
    g->pk = g->rank % Pz;
    CFLX_TRY(make_sub(c, g->pi * Py + g->pj, g->pk, Pz, &g->k_comm));
    return make_sub(c, g->pj * Pz + g->pk, g->pi, Px, &g->i_comm);
}
void grid_free(Grid* g) {
    for (SubComm* sc : {&g->k_comm, &g->i_comm})
        if (sc->c) ncclCommDestroy(sc->c);
}

int handle_init(Handle* h, const HandleTexts* texts, cflx_comm* c, int Px, int Py, int Pz) {
    h->texts = texts;
    CFLX_TRY(grid_init(h, c, Px, Py, Pz));
    CFLX_TRY(h->A0.alloc((size_t)h->Ml * h->Nl));
    return h->A11.alloc((size_t)h->Ml * h->Nl);
}
int handle_update_setup(Handle* h) {
    CFLX_TRY(gemm_tn_setup());
    // Trailing update: the FP64 DMMA kernel (gemm.cu).  On H100 the FP64 tensor rate (67 TFLOP/s) is above what the int8
    // digit-plane path can reach (989 int8 TMAC/s / 36 plane products = 55 TFLOP/s FP64-equivalent), so the int8 wgmma
    // path (ozaki.cu) runs only on request, CFLX_GEMM=ozaki, where the layer's contraction length is a whole number of
    // 128-element k chunks.
    const char* e = getenv("CFLX_GEMM");
    const bool int8 = e && !strcmp(e, "ozaki") && h->nlayr % 128 == 0 && h->nlayr <= 512;
    return h->update.create(h->Ml, h->Nl, h->nlayr, int8);
}
int handle_side_stream(Handle* h) {
    int lo = 0, hi = 0;
    cudaDeviceGetStreamPriorityRange(&lo, &hi);
    return h->side.create(cudaStreamNonBlocking, hi);
}
int handle_set_local(Handle* h, const double* host_local) {
    cudaStream_t s = h->comm->stream;
    CFLX_CUDA(cudaMemcpyAsync(h->A0, host_local, (size_t)h->Ml * h->Nl * sizeof(double), cudaMemcpyHostToDevice, s));
    CFLX_CUDA(cudaStreamSynchronize(s));
    h->have_input = true;
    h->factored = false;
    h->a0_is_next = false;
    h->sv.ready = false;
    h->eq.in.equed = 'N';
    return CFLX_OK;
}
int enter(Handle* h, const char* who, unsigned need) {
    const HandleTexts& t = *h->texts;
    char why[256] = "";
    if ((need & NEED_INPUT) && !h->have_input) snprintf(why, sizeof(why), "%s", t.no_input);
    else if ((need & NEED_UNSCALED) && h->eq.in.equed != 'N') snprintf(why, sizeof(why), t.scaled, h->eq.in.equed);
    else if ((need & NEED_FACTORS) && !h->factored) snprintf(why, sizeof(why), "%s", t.unfactored);
    else if ((need & NEED_OWN_INPUT) && h->a0_is_next)
        snprintf(why, sizeof(why), "refused: the input buffer of the last run was handed to the queued next matrix");
    else if ((need & NEED_FP64) && h->low_prec)
        snprintf(why, sizeof(why), "refused: the factors come from the TF32 trailing update of a mixed-precision driver, "
                                   "not from an FP64 factorisation; factor again first");
    if (why[0]) {
        set_last_error("%s: %s", who, why);
        return CFLX_ERR_STATE;
    }
    CFLX_CUDA(cudaSetDevice(h->comm->device));
    return CFLX_OK;
}
void handle_equil_begin(Handle* h) {
    h->factored = false;
    h->sv.ready = false;
}
int handle_equil_end(Handle* h, bool apply, int info, char equed, double rowcnd, double colcnd, const double* c) {
    if (apply && info == 0) CFLX_TRY(equil_record_set(&h->eq.in, equed, rowcnd, colcnd, h->eq.qr, c, h->M, h->comm->stream));
    return CFLX_OK;
}
int handle_launch_count(Handle* h, int64_t* count_out, int reset) {
    *count_out = h->launches;
    if (reset) h->launches = 0;
    return CFLX_OK;
}
}  // namespace cflx

namespace {
// One profiling region: always an NVTX range named like the reference's semiprof region; with profiling mode 1 a
// serialising CUDA-event timer (accurate per-phase device time, no overlap), with mode 2 an event pair on the launching
// stream that is resolved after the factorisation (no synchronisation: the timeline of the real, overlapped run).
struct PhaseTimer {
    cflx_lu* lu;
    int rg;
    cudaStream_t st;
    Events<2> ab;
    int ev = -1;
    PhaseTimer(cflx_lu* l, int region, cudaStream_t stream) : lu(l), rg(region), st(stream) {
        nvtxRangePushA(region_name(rg));
        if (lu->prof_mode == 1) {
            ab.create();
            cudaEventRecord(ab[0], st);
        } else if (lu->prof_mode == 2) {
            ev = (int)lu->tl_recs.size() * 2;
            while ((int)lu->tl_pool.size() < ev + 2) {
                lu->tl_pool.emplace_back();
                lu->tl_pool.back().create();
            }
            lu->tl_recs.push_back({rg, st == lu->comm->stream ? 0 : 1, ev});
            cudaEventRecord(lu->tl_pool[ev], st);
        }
    }
    ~PhaseTimer() {
        if (lu->prof_mode == 1) {
            cudaEventRecord(ab[1], st);
            cudaEventSynchronize(ab[1]);
            float ms = 0;
            cudaEventElapsedTime(&ms, ab[0], ab[1]);
            lu->phase_ms[region_phase(rg)] += ms;
            lu->region_ms[st == lu->comm->stream ? 0 : 1][rg] += ms;
            lu->region_cnt[st == lu->comm->stream ? 0 : 1][rg]++;
        } else if (lu->prof_mode == 2) {
            cudaEventRecord(lu->tl_pool[ev + 1], st);
        }
        nvtxRangePop();
    }
};

// exchange of tournament candidates with the butterfly partner(s) of round r (conflux_opt.hpp:242-280)
int tournament_exchange(cflx_lu* lu, int r, int my_half, cudaStream_t s) {
    const int v = lu->v, Px = lu->Px, pi = lu->pi;
    const int src = butterfly_pair(pi, r, Px);
    const int other = 1 - my_half;
    const size_t hv = (size_t)v * v;
    double* mine = lu->candH + my_half * hv;
    double* recv = lu->candH + other * hv;
    int* mine_t = lu->tagsH + my_half * v;
    int* recv_t = lu->tagsH + other * v;
    const bool self = (src == pi);
    if (self) {  // MPI_Sendrecv with itself: the own half is duplicated into the other half (conflux_opt.hpp:258-266)
        CFLX_CUDA(cudaMemcpyAsync(recv, mine, hv * sizeof(double), cudaMemcpyDeviceToDevice, s));
        CFLX_CUDA(cudaMemcpyAsync(recv_t, mine_t, v * sizeof(int), cudaMemcpyDeviceToDevice, s));
    }
    // a self-paired rank still serves one-sided requesters (the reference's extra Isend, conflux_opt.hpp:271-279)
    bool any = !self;
    for (int ppi = 0; ppi < Px && !any; ++ppi) any = (ppi != pi && butterfly_pair(ppi, r, Px) == pi);
    if (!any) return CFLX_OK;
    CFLX_NCCL(ncclGroupStart());
    for (int ppi = 0; ppi < Px; ++ppi) {
        if (ppi == pi || butterfly_pair(ppi, r, Px) != pi) continue;
        // mutual partner gets my own half; a one-sided requester gets the lower half
        const bool mutual = (!self && ppi == src);
        const double* sv = mutual ? mine : lu->candH + hv;
        const int* st = mutual ? mine_t : lu->tagsH + v;
        CFLX_NCCL(ncclSend(sv, hv, ncclDouble, ppi, lu->i_comm.c, s));
        CFLX_NCCL(ncclSend(st, v, ncclInt, ppi, lu->i_comm.c, s));
    }
    if (!self) {
        CFLX_NCCL(ncclRecv(recv, hv, ncclDouble, src, lu->i_comm.c, s));
        CFLX_NCCL(ncclRecv(recv_t, v, ncclInt, src, lu->i_comm.c, s));
    }
    CFLX_NCCL(ncclGroupEnd());
    return CFLX_OK;
}

// S[c][h*v + i] = candH[h][c][i]; tagsS likewise
__global__ void stack_kernel(const double* __restrict__ candH, const int* __restrict__ tagsH, int v, double* __restrict__ S,
                             double* __restrict__ W2, int* __restrict__ tagsS) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t tot = (int64_t)2 * v * v;
    if (e < tot) {
        const int c = (int)(e / (2 * v)), hi = (int)(e % (2 * v));
        const int h = hi / v, i = hi % v;
        const double x = candH[(size_t)h * v * v + (size_t)c * v + i];
        S[e] = x;
        W2[e] = x;
    }
    if (e < 2 * v) tagsS[e] = tagsH[e];
}

// ---- step 1 of iteration k in a prescribed row order (cflx_lu_factor_fixed), in place of the pivot search: the rows
// perm[kv, kv + v) located in this rank's panel and gathered (zeros for the rows other grid rows own), summed onto grid
// row k % Px (one contributor per element: the bits travel exactly as integers), and factored there without pivoting
// into A00 / A00T, with tagsH = the rows.  Everything after it in finish_step takes any v rows from any mix of ranks.
int fixed_panel(cflx_lu* lu, int k, int fnpr, int n_old, int64_t ldk, double* A00, double* A00T, cudaStream_t s) {
    const int v = lu->v, Px = lu->Px;
    const int* rows = lu->fix_perm + (size_t)k * v;
    {
        PhaseTimer t(lu, RG_step1_rowpermute, s);
        CFLX_TRY(launch_fixed_locate(rows, v, Px, lu->pi, fnpr, n_old, lu->igri, lu->perm, s));
        CFLX_TRY(launch_gather_winners(lu->PT, ldk, lu->gri + fnpr, n_old, lu->perm, v, lu->candH, v, lu->tagsS, 0, s));
        lu->launches += 2;
    }
    if (Px > 1) {
        PhaseTimer t(lu, RG_step1_pivoting, s);
        CFLX_NCCL(ncclReduce(lu->candH, lu->candH, (size_t)v * v, ncclUint64, ncclSum, k % Px, lu->i_comm.c, s));
    }
    if (lu->pi != k % Px) return CFLX_OK;
    PhaseTimer t(lu, RG_step1_lup, s);
    return launch_getrf_nopiv_tile(lu->candH, v, lu->fix_tiny, A00, A00T, rows, lu->tagsH, lu->fix_rec, k * v,
                                   getrf_nopiv_blocked(v), lu->fix_ws.p, s, &lu->launches);
}
// ---- steps 0 + 1 of iteration k: panel extract (+ layer reduce), local pivot search, tournament.  Runs on stream
// `s`; with look-ahead that is the high-priority side stream and overlaps the trailing update of iteration k-1.
// Touches only: PT, W, perm, candH/tagsH/S/W2/tagsS, A00/A00T (outputs consumed by finish_step(k) after the join).
int panel_phase(cflx_lu* lu, int k, int fnpr, cudaStream_t s) {
    const int v = lu->v, Px = lu->Px, Py = lu->Py, Pz = lu->Pz, Ml = lu->Ml, Nl = lu->Nl;
    const int pi = lu->pi, pj = lu->pj, pk = lu->pk;
    const int loff = (k / Py) * v, pjk = k % Py;
    if (pj != pjk) return CFLX_OK;
    // A00 / A00T are double-buffered by step parity: the look-ahead search of step k+1 must not overwrite the block
    // that the U solve and the factor stores of step k are still reading on the main stream
    double* A00 = lu->A00 + (size_t)(k & 1) * v * v;
    double* A00T = lu->A00T + (size_t)(k & 1) * v * v;
    const int n_old = Ml - fnpr;
    const int64_t ldk = std::max<int64_t>(2, round_up(n_old, 2));
    int nR = 0;
    while ((1 << nR) < Px) ++nR;
    // ---- step 0: panel extract (+ reduce over layers onto pk = 0)            conflux_opt.hpp:618-648
    {
        PhaseTimer t(lu, RG_step0_copy, s);
        CFLX_TRY(launch_extract_panel_T(lu->A11, Nl, fnpr, loff, n_old, v, lu->PT, ldk, s));
        lu->launches++;
    }
    if (Pz > 1 && n_old > 0) {
        PhaseTimer t(lu, RG_step0_reduce, s);
        CFLX_NCCL(ncclReduce(lu->PT, lu->PT, (size_t)v * ldk, ncclDouble, ncclSum, 0, lu->k_comm.c, s));
    }
    if (pk != 0) return CFLX_OK;
    if (lu->fixed) return fixed_panel(lu, k, fnpr, n_old, ldk, A00, A00T, s);
    // ---- step 1: local pivot search + tournament on column pj == k % Py, layer 0   conflux_opt.hpp:693-816
    int my_half = 0;
    {
        PhaseTimer t(lu, RG_step1_A10copy, s);
        CFLX_CUDA(cudaMemcpyAsync(lu->W, lu->PT, (size_t)v * ldk * sizeof(double), cudaMemcpyDeviceToDevice, s));
    }
    {
        PhaseTimer t(lu, RG_step1_lup, s);
        int nb_used = 0;
        if (nR == 0) {  // the local search already is the tournament: A00 comes from it (SURVEY.md fact 7)
            CFLX_TRY(launch_panel_getrf_a00(lu->W, ldk, n_old, v, lu->perm, A00, &nb_used, &lu->pws, s));
            CFLX_TRY(launch_gather_a00(lu->W, ldk, lu->perm, v, nb_used, A00, A00T, s));
            lu->launches += 2;
        } else {
            CFLX_TRY(launch_panel_getrf(lu->W, ldk, n_old, v, lu->perm, &lu->pws, s));
            lu->launches++;
        }
    }
    {
        PhaseTimer t(lu, RG_step1_rowpermute, s);
        int first_partner = flipbit(pi, 0);
        if (first_partner > Px - 1) first_partner = Px - 1;
        my_half = first_partner < pi ? 1 : 0;  // "higher rank puts his candidates below" (conflux_opt.hpp:717-750)
        CFLX_TRY(launch_gather_winners(lu->PT, ldk, lu->gri + fnpr, n_old, lu->perm, v,
                                       lu->candH + (size_t)my_half * v * v, v, lu->tagsH + my_half * v, 0, s));
        lu->launches++;
    }
    PhaseTimer t(lu, RG_step1_pivoting, s);
    for (int r = 0; r < nR; ++r) {
        CFLX_TRY(tournament_exchange(lu, r, my_half, s));
        const int64_t tot = (int64_t)2 * v * v;
        stack_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, s>>>(lu->candH, lu->tagsH, v, lu->S, lu->W2, lu->tagsS);
        CFLX_CUDA(cudaGetLastError());
        const bool last = (r == nR - 1);
        int nb_used = 0;
        if (last) {
            CFLX_TRY(launch_panel_getrf_a00(lu->W2, 2 * v, 2 * v, v, lu->perm, A00, &nb_used, &lu->pws, s));
            CFLX_TRY(launch_gather_a00(lu->W2, 2 * v, lu->perm, v, nb_used, A00, A00T, s));
            lu->launches++;
            my_half = 0;
        } else {
            CFLX_TRY(launch_panel_getrf(lu->W2, 2 * v, 2 * v, v, lu->perm, &lu->pws, s));
            my_half = butterfly_pair(pi, r + 1, Px) < pi ? 1 : 0;
        }
        CFLX_TRY(launch_gather_winners(lu->S, 2 * v, lu->tagsS, 2 * v, lu->perm, v, lu->candH + (size_t)my_half * v * v,
                                       v, lu->tagsH + my_half * v, 0, s));
        lu->launches += 3;
    }
    // winners now sit in the upper half: tagsH[0..v) = global pivot rows (conflux_opt.hpp:810-815)
    return CFLX_OK;
}

// the operands of this step's trailing update, split for a split kind: this layer's slab of L^T, and columns
// [col0, col0 + n) of its slab of U
int update_split_a(cflx_lu* lu, int n_act, int64_t ld2, cudaStream_t s) {
    if (!lu->update.splits() || n_act <= 0) return CFLX_OK;
    PhaseTimer t(lu, RG_step6_dgemm, s);
    lu->launches++;
    return lu->update.split_a(lu->LT + (int64_t)lu->pk * lu->nlayr * ld2, ld2, n_act, s);
}
int update_split_b(cflx_lu* lu, int col0, int n, int64_t ldu, cudaStream_t s) {
    if (!lu->update.splits() || n <= 0) return CFLX_OK;
    PhaseTimer t(lu, RG_step6_dgemm, s);
    lu->launches++;
    return lu->update.split_b(lu->U + (int64_t)lu->pk * lu->nlayr * ldu, ldu, col0, n, s);
}

int trailing_gemm(cflx_lu* lu, int k, int part, int fnpr, int n_act, int col_lo, int ncols, int64_t ld2, int64_t ldu,
                  int u_col_off, cudaStream_t s, int leave_sms = 0) {
    if (n_act <= 0 || ncols <= 0) return CFLX_OK;
    PhaseTimer t(lu, RG_step6_dgemm, s);
    GemmArgs g{};
    g.M = n_act;
    g.N = ncols;
    g.K = lu->nlayr;
    g.AT = lu->LT + (int64_t)lu->pk * lu->nlayr * ld2;
    g.ldat = ld2;
    g.B = lu->U + (int64_t)lu->pk * lu->nlayr * ldu + u_col_off;
    g.ldb = ldu;
    g.C = lu->A11 + (int64_t)fnpr * lu->Nl + col_lo;
    g.ldc = lu->Nl;
    g.D = lu->A11 + (int64_t)fnpr * lu->Nl + col_lo;
    g.ldd = lu->Nl;
    g.alpha = -1.0;
    g.beta = 1.0;
    const int e = 4 * k + 2 * part;
    if (lu->time_gemm) CFLX_CUDA(cudaEventRecord(lu->ev[e], s));
    CFLX_TRY(lu->update.apply(g, 0, u_col_off, leave_sms, s));
    if (lu->time_gemm) CFLX_CUDA(cudaEventRecord(lu->ev[e + 1], s));
    lu->ev_used[e / 2] = lu->time_gemm;
    lu->gemm_flops += 2.0 * g.M * (double)g.N * g.K;
    lu->launches++;
    return CFLX_OK;
}

// ---- everything of iteration k after the pivot search: pivot broadcast, row moves, solves, stores, trailing update
// (with the columns of panel k+1 updated first so that panel_phase(k+1) can start on the side stream).
int finish_step(cflx_lu* lu, int k, int& fnpr) {
    cudaStream_t s = lu->comm->stream;
    const int v = lu->v, Px = lu->Px, Py = lu->Py, Pz = lu->Pz, Ml = lu->Ml, Nl = lu->Nl;
    const int pi = lu->pi, pj = lu->pj, pk = lu->pk;
    const int loff = (k / Py) * v, pjk = k % Py, pik = k % Px;
    const bool on_col = (pj == pjk), on_row = (pi == pik), layer0 = (pk == 0);
    const int c0 = loff + (pj <= pjk ? v : 0);  // first live column of this rank after step k
    const int ncols = Nl - c0;
    const int fnpr_old = fnpr;
    const int n_old = Ml - fnpr_old;
    const int64_t ldk = std::max<int64_t>(2, round_up(n_old, 2));
    int nR = 0;
    while ((1 << nR) < Px) ++nR;
    double* A00 = lu->A00 + (size_t)(k & 1) * v * v;
    double* A00T = lu->A00T + (size_t)(k & 1) * v * v;
    // ---- A00 + pivot ids to everybody (one broadcast)                     conflux_opt.hpp:818-850,872
    {
        PhaseTimer t(lu, RG_step1_A00Buff_bcast, s);
        if (lu->P > 1) {
            const int root = (pik * Py + pjk) * Pz;  // rank of (k % Px, k % Py, 0)
            if (lu->rank == root) {
                CFLX_TRY(launch_pack_bcast(A00, lu->tagsH, v, lu->bcast, s));
                lu->launches++;
            }
            CFLX_NCCL(ncclBroadcast(lu->bcast, lu->bcast, (size_t)v * v + v, ncclDouble, root, lu->comm->world, s));
            CFLX_TRY(launch_unpack_bcast(lu->bcast, v, A00, A00T, lu->gpivots, s));
            lu->launches++;
        } else {
            CFLX_CUDA(cudaMemcpyAsync(lu->gpivots, lu->tagsH, v * sizeof(int), cudaMemcpyDeviceToDevice, s));
        }
        CFLX_TRY(launch_record_pivots(lu->gpivots, v, lu->hist, k, s));
        lu->launches++;
    }
    // ---- step 2: localise pivots, push them up, extract pivot rows        conflux_opt.hpp:876-1147
    // At Px > 1 the host needs this rank's pivot count (it sizes the L-panel work).  Everything that does NOT depend
    // on it -- row moves, pivot-row reduce, the U solve, its broadcast, the factor stores -- is enqueued first, and
    // the host only then waits for the 4-byte read-back, so the GPU stays busy while the rest is enqueued.
    {
        PhaseTimer t(lu, RG_step2_pushingpivots, s);
        CFLX_TRY(launch_plan_moves(lu->gpivots, v, Px, pi, fnpr_old, Ml, lu->igri, lu->plan, s));
        lu->launches++;
        if (Px > 1 && !lu->fixed) {  // a prescribed order gives the count on the host
            CFLX_CUDA(cudaMemcpyAsync(lu->h_npiv, lu->plan.npiv, sizeof(int), cudaMemcpyDeviceToHost, s));
            CFLX_CUDA(cudaEventRecord(lu->ev_npiv, s));
        }
        const int col_lo = layer0 ? 0 : loff;
        const int64_t ldu0 = std::max(2, ncols);
        CFLX_TRY(launch_push_phase1(lu->A11, Nl, Nl, col_lo, lu->plan, v, lu->tmp, ncols > 0 ? lu->A01raw.p : nullptr, ldu0,
                                    c0, s));
        CFLX_TRY(launch_push_phase2(lu->A11, Nl, Nl, col_lo, lu->plan, v, s));
        CFLX_TRY(launch_push_phase3(lu->A11, Nl, Nl, col_lo, fnpr_old, lu->plan, v, lu->tmp, s));
        CFLX_TRY(launch_update_gri(lu->gri, lu->gri_tmp, lu->igri, lu->plan.rowsrc, fnpr_old, Ml, v, Px, s));
        lu->launches += 5;
    }
    const int64_t ldu = std::max(2, ncols);
    // At Px == 1 the local pivot search IS the panel factorisation: its multipliers are the L panel (same values a
    // LAPACK getrf leaves behind; the reference recomputes them with dtrsm against A00, conflux_opt.hpp:1347).  A
    // prescribed order has no panel factorisation: L comes from the TRSM, as on Px > 1 grids.
    const bool fused_l = (nR == 0) && !lu->fixed;
    // ---- steps 2b/3: pivot rows summed over layers and gathered on row pi == k % Px   conflux_opt.hpp:1164-1260
    if (ncols > 0 && Px * Pz > 1) {
        PhaseTimer t(lu, RG_step2_reduce, s);
        CFLX_NCCL(ncclReduce(lu->A01raw, lu->A01raw, (size_t)v * ldu, ncclDouble, ncclSum, pik * Pz, lu->ik_comm.c, s));
    }
    // ---- step 5 first: U = L00^-1 * (pivot rows)                            conflux_opt.hpp:1522-1593
    if (layer0 && ((on_col && !fused_l) || on_row)) {
        PhaseTimer t(lu, RG_step5_dtrsm, s);
        CFLX_TRY(launch_diag_inverses(A00, v, lu->nb, lu->Uinv, lu->LinvT, s));
        lu->launches++;
    }
    // The U solve is split in two column windows: the first v columns (= the next panel) are solved before the
    // look-ahead fork, the rest after it, off the pivot search's critical path (single-rank grids only: with more
    // ranks the U panel is broadcast whole).
    const bool split_u = (lu->P == 1) && (k + 1 < lu->Nt) && ncols > v;
    const int ncols_a = split_u ? v : ncols;
    if (on_row && layer0 && ncols > 0) {
        PhaseTimer t(lu, RG_step5_dtrsm, s);
        CFLX_TRY(trsm_left_lower_unit(A00T, lu->LinvT, v, lu->nb, lu->A01raw, lu->U, ldu, ncols_a, s));
        lu->launches += 2 * (v / lu->nb) - 1;
    }
    if (Px * Pz > 1 && ncols > 0) {  // U panel to every (pi', pk') of my grid column   conflux_opt.hpp:1567-1593
        PhaseTimer t(lu, RG_step5_comm, s);
        CFLX_NCCL(ncclBroadcast(lu->U, lu->U, (size_t)v * ldu, ncclDouble, pik * Pz, lu->ik_comm.c, s));
    }
    auto store_factors = [&]() -> int {  // my promoted rows receive their U part and diagonal block   :1721-1754
        if (!layer0) return CFLX_OK;
        PhaseTimer t(lu, RG_storingresults, s);
        if (ncols > 0) {
            CFLX_TRY(launch_store_u_rows(lu->A11, Nl, fnpr_old, lu->plan, lu->U, ldu, c0, ncols, v, s));
            lu->launches++;
        }
        if (on_col) {
            CFLX_TRY(launch_store_diag(lu->A11, Nl, fnpr_old, lu->plan, A00, loff, v, s));
            lu->launches++;
        }
        return CFLX_OK;
    };
    if (!split_u) CFLX_TRY(store_factors());
    // ---- now the pivot count: sizes of the L panel and of the trailing update
    int npiv = v;
    if (lu->fixed) {
        npiv = lu->fix_npiv[k];
    } else if (Px > 1) {
        CFLX_CUDA(cudaEventSynchronize(lu->ev_npiv));
        npiv = *lu->h_npiv;
    }
    if (npiv < 0 || npiv > v || fnpr_old + npiv > Ml) {
        set_last_error("step %d: inconsistent pivot count %d (fnpr %d, Ml %d)", k, npiv, fnpr_old, Ml);
        return CFLX_ERR_STATE;
    }
    fnpr = fnpr_old + npiv;
    const int n_act = Ml - fnpr;
    const int64_t ld2 = std::max<int64_t>(2, round_up(n_act, 2));
    // ---- step 4: L = A10 * U00^-1 on the panel column                       conflux_opt.hpp:1329-1434
    if (on_col && layer0 && n_act > 0) {
        {
            PhaseTimer t(lu, RG_step4_reshuffling, s);
            CFLX_TRY(launch_compact_panel(fused_l ? lu->W : lu->PT, ldk, fused_l ? lu->LT : lu->PT2, ld2, lu->plan.rowsrc,
                                          fnpr_old, lu->plan.npiv, Ml, v, s));
            lu->launches++;
        }
        if (!fused_l) {
            PhaseTimer t(lu, RG_step4_dtrsm, s);
            CFLX_TRY(trsm_right_upper_T(A00, lu->Uinv, v, lu->nb, lu->PT2, lu->LT, ld2, n_act, s));
            lu->launches += 2 * (v / lu->nb) - 1;
        }
        PhaseTimer t(lu, RG_storingresults, s);
        CFLX_TRY(launch_store_panel_T(lu->A11, Nl, fnpr, loff, n_act, v, lu->LT, ld2, s));  // L in place
        lu->launches++;
    }
    if (Py * Pz > 1 && n_act > 0) {  // L panel to every (pj', pk') of my grid row    conflux_opt.hpp:1404-1434
        PhaseTimer t(lu, RG_step4_comm, s);
        CFLX_NCCL(ncclBroadcast(lu->LT, lu->LT, (size_t)v * ld2, ncclDouble, pjk * Pz, lu->jk_comm.c, s));
    }
    // ---- step 6: trailing update on every rank and layer                    conflux_opt.hpp:1628-1632
    // Look-ahead: the rank that owns panel k+1 updates those v columns first (they are its first live block), forks
    // the pivot search of iteration k+1 onto the side stream, and only then updates the remaining columns.
    const bool next_col = (k + 1 < lu->Nt) && (pj == (k + 1) % Py);
    CFLX_TRY(update_split_a(lu, n_act, ld2, s));
    if (n_act > 0) CFLX_TRY(update_split_b(lu, 0, split_u ? std::min(v, ncols) : ncols, ldu, s));
    if (next_col) {
        const int w = std::min(v, ncols);
        CFLX_TRY(trailing_gemm(lu, k, 0, fnpr, n_act, c0, w, ld2, ldu, 0, s));
        cudaStream_t side = (lu->prof_mode == 1) ? nullptr : lu->side.s;  // phase profiling serialises everything
        cudaStream_t sp = side ? side : s;
        if (side) {
            CFLX_CUDA(cudaEventRecord(lu->ev_fork, s));
            CFLX_CUDA(cudaStreamWaitEvent(sp, lu->ev_fork, 0));
        }
        CFLX_TRY(panel_phase(lu, k + 1, fnpr, sp));
        if (side) CFLX_CUDA(cudaEventRecord(lu->ev_join, sp));
        if (split_u) {
            PhaseTimer t(lu, RG_step5_dtrsm, s);
            CFLX_TRY(trsm_left_lower_unit(A00T, lu->LinvT, v, lu->nb, lu->A01raw + v, lu->U + v, ldu, ncols - v, s));
            lu->launches += 2 * (v / lu->nb) - 1;
        }
        if (split_u) CFLX_TRY(store_factors());
        if (split_u && n_act > 0) CFLX_TRY(update_split_b(lu, w, ncols - w, ldu, s));
        // the persistent split kernels leave the SMs of the concurrent pivot search alone
        CFLX_TRY(trailing_gemm(lu, k, 1, fnpr, n_act, c0 + w, ncols - w, ld2, ldu, w, s, side ? lu->pws.cta_cap : 0));
        if (side) CFLX_CUDA(cudaStreamWaitEvent(s, lu->ev_join, 0));
    } else {
        CFLX_TRY(trailing_gemm(lu, k, 0, fnpr, n_act, c0, ncols, ld2, ldu, 0, s));
    }
    return CFLX_OK;
}

// ---------------------------------------------------------------------------------------------- solve, A X = B
// The factors in the conflux layout of the validation path (Cbuf, as cflx_lu_get_factors leaves them), described to the
// solve engine (solve.cu).  Every layer joins the grid-row reduces and grid-column broadcasts (jk / ik communicators,
// layer 0 at rank p * Pz), the layers pk != 0 with zeros.
SolveFactor lu_solve_factor(cflx_lu* lu) { return SolveFactor{*lu, lu->Cbuf, lu->Ml, &lu->jk_comm, &lu->ik_comm, lu->Pz}; }

// *perm = the permutation of the last factorisation (M ints), in stream order
int lu_permutation(cflx_lu* lu, std::vector<int>* perm) {
    perm->resize(lu->M);
    CFLX_CUDA(cudaMemcpyAsync(perm->data(), lu->hist, sizeof(int) * lu->M, cudaMemcpyDeviceToHost, lu->comm->stream));
    CFLX_CUDA(cudaStreamSynchronize(lu->comm->stream));
    return CFLX_OK;
}

// First call after a factorisation: the factors redistributed into Cbuf, the diagonal-block inverses, and on the ranks
// that seed the right-hand side, the row of B that each local row of P*B comes from.
int lu_solve_prepare(cflx_lu* lu) {
    cudaStream_t s = lu->comm->stream;
    const int v = lu->v, Px = lu->Px, Ml = lu->Ml;
    std::vector<int> hist;
    CFLX_TRY(lu_permutation(lu, &hist));
    if (lu->pk == 0) {
        lu->sv.inv.reset();  // before the redistribution allocates its staging
        if (!lu->Cbuf) CFLX_TRY(lu->Cbuf.alloc((size_t)Ml * lu->Nl));
        int rc = redistribute_pivoted_rows(lu, hist, true, lu->A11, lu->Cbuf);
        lu->xbuf.reset();  // 2 x local matrix of staging: do not keep it alive
        if (rc) return rc;
        CFLX_TRY(solve_inverses(&lu->sv, lu_solve_factor(lu), false));
        if (lu->pj == 0) {  // local row (k / Px)*v + i of P*B is row hist[k*v + i] of B, for the tiles k of this grid row
            std::vector<int> rows(Ml, 0);
            for (int q = 0; q < lu->M; ++q) {
                const int k = q / v;
                if (k % Px == lu->pi) rows[(k / Px) * v + q % v] = hist[q];
            }
            CFLX_TRY(solve_set_rows(&lu->sv.rows, rows, s));
        }
    }
    lu->sv.ready = true;
    lu->sv.trans_ready = false;
    return CFLX_OK;
}

// First transposed solve or condition estimate after a factorisation: the seeding maps of P*A solved without P (B by
// local tile row on the ranks (pi, 0, 0) and by local tile column on the ranks (0, pj, 0), identity in both), and on every
// rank the inverse permutation that puts W[q] at row perm[q] of X.
int lu_solve_prepare_trans(cflx_lu* lu) {
    cudaStream_t s = lu->comm->stream;
    const int v = lu->v, Px = lu->Px, Py = lu->Py;
    std::vector<int> hist;
    CFLX_TRY(lu_permutation(lu, &hist));
    std::vector<int> unperm(lu->M);
    for (int q = 0; q < lu->M; ++q) unperm[hist[q]] = q;
    CFLX_TRY(solve_set_rows(&lu->sv.unperm, unperm, s));
    if (lu->pk == 0 && lu->pj == 0) {
        std::vector<int> rows(lu->Ml, 0);
        for (int q = 0; q < lu->M; ++q)
            if ((q / v) % Px == lu->pi) rows[(q / v / Px) * v + q % v] = q;
        CFLX_TRY(solve_set_rows(&lu->sv.rows_id, rows, s));
    }
    if (lu->pk == 0 && lu->pi == 0) {
        std::vector<int> cols(lu->Nl, 0);
        for (int q = 0; q < lu->M; ++q)
            if ((q / v) % Py == lu->pj) cols[(q / v / Py) * v + q % v] = q;
        CFLX_TRY(solve_set_rows(&lu->sv.cols, cols, s));
    }
    lu->sv.trans_ready = true;
    return CFLX_OK;
}

// One solve with the factors of the last factorisation.  transposed: A^T X = B, else A X = B.  pa: the system is P*A
// (no row map of B in A X = B, no final P^T in A^T X = B), as the condition estimate runs it.  X may be null (the solved
// system then stays in lu->sv.X, or sv.Xg after P^T).
int lu_sweeps(cflx_lu* lu, bool transposed, bool pa, int nrhs, const double* B, int ldb, double* X, int ldx) {
    if (!lu->sv.ready) CFLX_TRY(lu_solve_prepare(lu));
    if ((transposed || pa) && !lu->sv.trans_ready) CFLX_TRY(lu_solve_prepare_trans(lu));
    const SolveFactor f = lu_solve_factor(lu);
    SolveCache* sc = &lu->sv;
    const int ldn = (int)round_up(nrhs, 8);
    CFLX_TRY(solve_cache_grow(sc, f, ldn, true, transposed, transposed));
    if (!transposed) {
        CFLX_TRY(solve_seed(sc, f, ldn, nrhs, B, ldb, SolveSeed{false, pa ? sc->rows_id : sc->rows, lu->Ml, sc->W}));
        // L Y = P B keeping Y_t as the owner's W rows, so that U X = Y starts from W = Y
        CFLX_TRY(solve_row_sweep(sc, f, ldn, true, sc->W, lu->Px, true));
        CFLX_TRY(solve_row_sweep(sc, f, ldn, false, sc->X, 1, false));
        return solve_finish(sc, f, ldn, nrhs, X, ldx);
    }
    // A^T X = B <=> U^T (L^T W) = B, X[perm[q]] = W[q]: U^T Y = B keeping Y_t as the owner's Z columns, so that L^T W = Y
    // starts from Z = Y
    CFLX_TRY(solve_seed(sc, f, ldn, nrhs, B, ldb, SolveSeed{true, sc->cols, lu->Nl, sc->Z}));
    CFLX_TRY(solve_col_sweep(sc, f, ldn, true, Tri::UpperT, sc->Z, lu->Py, true));
    CFLX_TRY(solve_col_sweep(sc, f, ldn, false, Tri::UnitLowerT, sc->X, 1, false));
    return solve_finish(sc, f, ldn, nrhs, X, ldx, pa ? nullptr : sc->unperm.p);
}

const HandleTexts kLuTexts = {
    "requested before cflx_lu_factor, or after cflx_lu_set_local without a factorisation",
    "requested before cflx_lu_set_local",
    "refused: the input is already scaled (equed = '%c'); upload it again first"};

// LAPACK dgecon on the grid, NORM = '1' or (inf) 'I': the norm of the input A0 (the padded M x M matrix), and the
// Hager-Higham estimate of ||inv(P A)||_1 = ||inv(A)||_1 from inv(U) inv(L) x and inv(L)^T inv(U)^T x, as dgecon runs it
// on L and U alone; ||inv(A)||_inf is the same estimate with the two kinds of product swapped.
int lu_rcond(cflx_lu* lu, bool inf, double* rcond_out, double* anorm_out) {
    double anorm = 0.0, ainvnm = 0.0;
    CFLX_TRY(inf ? norminf_grid(*lu, lu->A0, &anorm) : norm1_grid(*lu, lu->A0, false, &anorm));
    if (anorm > 0.0) {
        // every rank runs the estimator on the X of solve_finish, bit-identical on every rank, so every rank makes the
        // same choices and issues the same solves (the same collectives) in the same order
        auto apply = [&](int kase, double* x) { return lu_sweeps(lu, (kase == 2) != inf, true, 1, x, 1, x, 1); };
        CFLX_TRY(estimate_inv_norm1(lu->M, apply, &ainvnm));
    }
    *rcond_out = rcond_from(anorm, ainvnm);
    if (anorm_out) *anorm_out = anorm;
    return CFLX_OK;
}

// dgerfs on the input A0 with the solves above.  For trans = 0 the estimator's kase 1 (inv(A)^T) is the transposed solve
// and kase 2 the plain one; for trans = 1 they swap.
RefineOp lu_refine_op(cflx_lu* lu, bool t) {
    auto solve = [lu, t](bool tk, int n, const double* b, int lb, double* x, int lx) {
        return lu_sweeps(lu, t != tk, false, n, b, lb, x, lx);
    };
    return RefineOp{*lu, lu->A0, t ? ResidMode::TN : ResidMode::NN, false, solve};
}

// What refine_x, svx and svxx compute of the matrix, once per call whatever the right-hand sides: the first exactly zero
// U(k,k) over the world (with rpvgrw set, through the pivot growth: dla_gerpvgrw when per_column, else dgesvx's), then,
// when there is none, dgecon in the infinity-norm (inf) or the 1-norm; rcond is 0 when there is one.
int lu_expert_pre(cflx_lu* lu, bool inf, double* rpvgrw, bool per_column, double* rcond, int* info) {
    if (!lu->sv.ready) CFLX_TRY(lu_solve_prepare(lu));
    *rcond = 0.0;
    if (rpvgrw) CFLX_TRY(pivot_growth_grid(*lu, &lu->eq, lu->Cbuf, lu->A0, per_column, rpvgrw, info));
    else CFLX_TRY(zero_pivot_grid(*lu, &lu->eq, lu->Cbuf, info));
    return *info > 0 ? CFLX_OK : lu_rcond(lu, inf, rcond, nullptr);
}

// The scales of op(A) X = B the factors carry: pre for the rows of B (r for trans 0, c for trans 1; null when the
// factors carry none), post for the rows of X and the error bounds' d (the other one), cnd the ratio that divides ferr.
struct LuScales {
    const double *pre, *post;
    double cnd;
};
LuScales lu_scales(const cflx_lu* lu, bool t) {
    const EquilRecord& eq = lu->eq.fac;
    const double* r = eq.equed == 'R' || eq.equed == 'B' ? eq.r.p : nullptr;
    const double* c = eq.equed == 'C' || eq.equed == 'B' ? eq.c.p : nullptr;
    return LuScales{t ? c : r, t ? r : c, t ? eq.rowcnd : eq.colcnd};
}

// cflx_lu_equilibrate (dgeequ) and, with pow2, cflx_lu_equilibrate_b (dgeequb), as `who`
int lu_equilibrate(const char* who, cflx_lu* lu, int apply, bool pow2, double* r_out, double* c_out, double* rowcnd_out,
                   double* colcnd_out, double* amax_out, char* equed_out, int* info_out) {
    REFUSE_FOR(who, !lu);
    REFUSE_FOR(who, apply != 0 && apply != 1);
    REFUSE_FOR(who, !info_out);
    if (apply && lu->rbt.in.depth) {
        set_last_error("%s: refused, the input carries a random butterfly transform (cflx_lu_rbt); upload it again first",
                       who);
        return CFLX_ERR_STATE;
    }
    CFLX_TRY(enter(lu, who, NEED_INPUT | (apply ? NEED_UNSCALED : 0u)));
    handle_equil_begin(lu);
    if (lu->a0_is_next) CFLX_CUDA(cudaStreamWaitEvent(lu->comm->stream, lu->ev_upload, 0));  // A0 holds a streamed next input
    double rowcnd = 0.0, colcnd = 0.0, amax = 0.0;
    char equed = 'N';
    int info = 0;
    CFLX_TRY(geequ_grid(*lu, &lu->eq, lu->A0, apply != 0, pow2, r_out, c_out, &rowcnd, &colcnd, &amax, &equed, &info));
    CFLX_TRY(handle_equil_end(lu, apply != 0, info, equed, rowcnd, colcnd, lu->eq.qc));
    if (rowcnd_out) *rowcnd_out = rowcnd;
    if (colcnd_out) *colcnd_out = colcnd;
    if (amax_out) *amax_out = amax;
    if (equed_out) *equed_out = equed;
    *info_out = info;
    return CFLX_OK;
}

// cflx_lu_validate as `who`
int lu_validate(const char* who, cflx_lu* lu, double* abs_out, double* rel_out) {
    CFLX_TRY(enter(lu, who, NEED_FACTORS | NEED_OWN_INPUT));
    std::vector<int> hist;
    CFLX_TRY(lu_permutation(lu, &hist));
    return lu_residual_grid(lu, hist, abs_out, rel_out);
}

// the visible CUDA devices (0 when the runtime finds none)
int device_count() {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        n = 0;
        cudaGetLastError();
    }
    return n;
}

// lu_params::get_p_grid (lu_params.hpp:21-47) for M, N, P >= 1
void auto_grid(int M, int N, int P, int* Px, int* Py, int* Pz) {
    const double ratio = 1.0 * std::max(M, N) / std::min(M, N);
    const int p1 = (int)std::cbrt(P / ratio);
    const int psq = (int)std::sqrt(P / ratio);
    const int phs = (int)std::sqrt(P / (2 * ratio));
    if (P == psq * psq) {
        *Px = psq; *Py = psq; *Pz = 1;
        return;
    }
    if (phs * phs == P / 2) {
        *Px = phs; *Py = phs; *Pz = 2;
        return;
    }
    int d[3] = {p1, (int)(ratio * p1), 0};
    d[2] = P / (d[0] * d[1]);
    std::sort(d, d + 3, [](int a, int b) { return a > b; });
    *Px = d[0]; *Py = d[1]; *Pz = d[2];
}

// lu_params::initialize's sizes (lu_params.hpp:67-82) into o[8] (cflx_lu_dims), refused in the name of `who`
int lu_dims(const char* who, int M, int N, int v, int Px, int Py, int Pz, int* o) {
    REFUSE_FOR(who, M <= 0);
    REFUSE_FOR(who, N <= 0);
    REFUSE_FOR(who, v <= 0);
    REFUSE_FOR(who, Px <= 0);
    REFUSE_FOR(who, Py <= 0);
    REFUSE_FOR(who, Pz <= 0);
    const int tx = (int)std::ceil((double)M / (v * Px)), ty = (int)std::ceil((double)N / (v * Py));
    const int Mp = v * Px * tx, Np = v * Py * ty;
    const int Nt = (int)std::ceil((double)Np / v), Mt = (int)std::ceil((double)Mp / v);
    o[0] = Mp; o[1] = Np;
    o[2] = (int)std::ceil((double)Mt / Px) * v;
    o[3] = (int)std::ceil((double)Nt / Py) * v;
    o[4] = Nt; o[5] = (v + Pz - 1) / Pz; o[6] = Mt; o[7] = Px * Py * Pz;
    return CFLX_OK;
}
}  // namespace

// ======================================================================================================== C ABI
extern "C" {

const char* cflx_last_error(void) { return g_err; }
const char* cflx_version(void) { return "conflux_b200 0.1 (sm_90a)"; }

int cflx_device_count(int* count) {
    *count = device_count();
    return CFLX_OK;
}

int cflx_get_unique_id(void* id_out) {
    static_assert(sizeof(ncclUniqueId) == CFLX_UNIQUE_ID_BYTES, "unique id size");
    ncclUniqueId id;
    CFLX_NCCL(ncclGetUniqueId(&id));
    std::memcpy(id_out, &id, sizeof(id));
    return CFLX_OK;
}

int cflx_comm_create(int world_size, int world_rank, const void* unique_id, int device, cflx_comm** out) {
    REFUSE_IF(!out);
    REFUSE_IF(world_size < 1);
    REFUSE_IF(world_rank < 0);
    REFUSE_IF(world_rank >= world_size);
    const int ndev = device_count();
    if (ndev == 0) {
        set_last_error("%s: no CUDA device visible: conflux_b200 has no CPU fallback", __func__);
        return CFLX_ERR_NO_DEVICE;
    }
    if (device < 0 || device >= ndev) {
        set_last_error("%s: device %d out of range (%d visible)", __func__, device, ndev);
        return CFLX_ERR_ARG;
    }
    CFLX_CUDA(cudaSetDevice(device));
    std::unique_ptr<cflx_comm> c(new cflx_comm);
    c->world_size = world_size;
    c->world_rank = world_rank;
    c->device = device;
    CFLX_TRY(c->stream.create(cudaStreamNonBlocking));
    CFLX_TRY(c->d_scratch.alloc_exact(1));
    CFLX_CUDA(cudaMemset(c->d_scratch, 0, sizeof(double)));
    if (world_size > 1) {
        REFUSE_IF(!unique_id);
        ncclUniqueId id;
        std::memcpy(&id, unique_id, sizeof(id));
        CFLX_NCCL(ncclCommInitRank(&c->world, world_size, id, world_rank));
    }
    *out = c.release();
    return CFLX_OK;
}

int cflx_comm_barrier(cflx_comm* c) {
    REFUSE_IF(!c);
    CFLX_CUDA(cudaSetDevice(c->device));
    return grid_barrier(c);
}

void cflx_comm_destroy(cflx_comm* c) {
    if (!c) return;
    cudaSetDevice(c->device);
    if (c->world) ncclCommDestroy(c->world);
    delete c;
}

int cflx_auto_grid(int M, int N, int P, int* Px, int* Py, int* Pz) {
    REFUSE_IF(M <= 0);
    REFUSE_IF(N <= 0);
    REFUSE_IF(P <= 0);
    auto_grid(M, N, P, Px, Py, Pz);
    return CFLX_OK;
}

int cflx_lu_dims(int M, int N, int v, int Px, int Py, int Pz, int* o) {
    REFUSE_IF(!o);
    return lu_dims(__func__, M, N, v, Px, Py, Pz, o);
}

int cflx_init_matrix_host(int M, int N, int v, int Px, int Py, int Pz, int rank, int seed, double* out) {
    int d[8];
    CFLX_TRY(lu_dims(__func__, M, N, v, Px, Py, Pz, d));
    const int Ml = d[2], Nl = d[3];
    REFUSE_IF(rank < 0);
    REFUSE_IF(rank >= Px * Py * Pz);
    REFUSE_IF(!out);
    std::fill(out, out + (size_t)Ml * Nl, 0.0);
    if (rank % Pz != 0) return CFLX_OK;  // layers pk != 0 start at zero (lu_params.hpp:149-155)
    // lu_params.hpp:157-363: for (padded) M == N in {8, 9, 16, 20, 27, 32} the reference fills a FIXED matrix,
    // element (gi, gj) of the table at the tile-layout slot of this rank
    if (d[0] == d[1]) {
        std::vector<double> tab;
        if (fixed_input_matrix(d[0], &tab)) {
            const int n = d[0];
            const Layout L{n, v, d[4], Ml, Nl, Px, Py, rank / (Py * Pz), (rank / Pz) % Py};
            for (int lr = 0; lr < Ml; ++lr)
                for (int lc = 0; lc < Nl; ++lc) out[(size_t)lr * Nl + lc] = tab[(size_t)L.row(lr) * n + L.col(lc)];
            return CFLX_OK;
        }
    }
    // lu_params.hpp:364-375: mt19937_64(seed + rank), values 5 + U[0,1), tile by tile (lti outer, ltj inner),
    // row-major inside a tile (libs/costa/src/costa/grid2grid/grid_layout.hpp:68-92)
    std::mt19937_64 eng((unsigned long long)(seed + rank));
    std::uniform_real_distribution<double> dist;
    for (int lti = 0; lti < Ml / v; ++lti)
        for (int ltj = 0; ltj < Nl / v; ++ltj)
            for (int li = 0; li < v; ++li)
                for (int lj = 0; lj < v; ++lj) out[(size_t)(lti * v + li) * Nl + ltj * v + lj] = 5 + dist(eng);
    return CFLX_OK;
}

int cflx_lu_create(cflx_comm* c, int M, int N, int v, int Px, int Py, int Pz, cflx_lu** out) {
    REFUSE_IF(!c);
    REFUSE_IF(!out);
    REFUSE_IF(M <= 0);
    REFUSE_IF(N <= 0);
    REFUSE_IF(v <= 0);
    CFLX_CUDA(cudaSetDevice(c->device));
    if (Px <= 0 || Py <= 0 || Pz <= 0) auto_grid(M, N, c->world_size, &Px, &Py, &Pz);
    if (Px != Py) {
        set_last_error("%s: grid %dx%dx%d: the CONFLUX LU path requires Px == Py (SURVEY.md fact 6)", __func__, Px, Py, Pz);
        return CFLX_ERR_UNSUPPORTED;
    }
    if (Px * Py * Pz != c->world_size) {
        set_last_error("%s: grid %dx%dx%d does not match the %d ranks of the communicator", __func__, Px, Py, Pz,
                       c->world_size);
        return CFLX_ERR_ARG;
    }
    if (v % 4 != 0 || v % Pz != 0 || (v / Pz) % 4 != 0 || pick_nb(v) == 0) {
        set_last_error("%s: tile size v=%d unsupported: need v %% 4 == 0 and (v / Pz) %% 4 == 0", __func__, v);
        return CFLX_ERR_UNSUPPORTED;
    }
    int d[8];
    CFLX_TRY(lu_dims(__func__, M, N, v, Px, Py, Pz, d));
    if (d[0] != d[1]) {
        set_last_error("%s: only square matrices are supported (the miniapp passes M = N)", __func__);
        return CFLX_ERR_UNSUPPORTED;
    }
    std::unique_ptr<cflx_lu> lu(new cflx_lu);
    lu->M = d[0]; lu->N = d[1]; lu->Ml = d[2]; lu->Nl = d[3]; lu->Nt = d[4]; lu->nlayr = d[5]; lu->Mt = d[6];
    lu->v = v;
    lu->nb = pick_nb(v);
    // sub-communicators (all ranks call all splits, same order)
    CFLX_TRY(handle_init(lu.get(), &kLuTexts, c, Px, Py, Pz));
    CFLX_TRY(make_sub(c, lu->pi, lu->pj * Pz + lu->pk, Py * Pz, &lu->jk_comm));
    CFLX_TRY(make_sub(c, lu->pj, lu->pi * Pz + lu->pk, Px * Pz, &lu->ik_comm));

    const int64_t ldp = round_up(lu->Ml, 2) + 2;
    lu->ldp_max = ldp;
    const size_t pan = (size_t)v * ldp, upan = (size_t)v * (lu->Nl + 2), vv = (size_t)v * v;
    CFLX_TRY(lu->PT.alloc(pan)); CFLX_TRY(lu->PT2.alloc(pan)); CFLX_TRY(lu->W.alloc(pan)); CFLX_TRY(lu->LT.alloc(pan));
    CFLX_TRY(lu->A01raw.alloc(upan)); CFLX_TRY(lu->U.alloc(upan)); CFLX_TRY(lu->tmp.alloc((size_t)v * lu->Nl));
    CFLX_TRY(lu->A00.alloc(2 * vv)); CFLX_TRY(lu->A00T.alloc(2 * vv)); CFLX_TRY(lu->Uinv.alloc(vv));
    CFLX_TRY(lu->LinvT.alloc(vv)); CFLX_TRY(lu->candH.alloc(2 * vv)); CFLX_TRY(lu->S.alloc(2 * vv));
    CFLX_TRY(lu->W2.alloc(2 * vv)); CFLX_TRY(lu->bcast.alloc(vv + v));
    CFLX_TRY(lu->gri.alloc(lu->Ml)); CFLX_TRY(lu->gri_tmp.alloc(lu->Ml)); CFLX_TRY(lu->igri.alloc(lu->Ml));
    CFLX_TRY(lu->perm.alloc(2 * v)); CFLX_TRY(lu->gpivots.alloc(v)); CFLX_TRY(lu->tagsH.alloc(2 * v));
    CFLX_TRY(lu->tagsS.alloc(2 * v)); CFLX_TRY(lu->hist.alloc(lu->M));
    CFLX_TRY(lu->plan_mem.alloc(6 * (size_t)v + 8 + lu->Ml));
    int* pm = lu->plan_mem;
    lu->plan.npiv = pm; lu->plan.nel = pm + 4; pm += 8;
    lu->plan.cur_piv = pm; pm += v;
    lu->plan.order = pm; pm += v;
    lu->plan.slot2piv = pm; pm += v;
    lu->plan.early = pm; pm += v;
    lu->plan.late = pm; pm += v;
    pm += v;
    lu->plan.rowsrc = pm;
    CFLX_TRY(lu->h_npiv.alloc(1));
    CFLX_TRY(lu->ev_npiv.create(cudaEventDisableTiming));
    CFLX_TRY(panel_workspace_create(&lu->pws));
    CFLX_TRY(handle_update_setup(lu.get()));
    {
        // look-ahead: pivot search of iteration k+1 (extract, layer reduce, local search, tournament exchanges) on a
        // high-priority side stream, on a capped number of SMs, while the trailing update of iteration k runs on the
        // rest.  A rank never has NCCL work in flight on both streams: the side stream's collectives (k- and
        // i-communicator) sit between the fork after GEMM_next and the join before the next world broadcast.
        const char* e = getenv("CFLX_LOOKAHEAD");
        const char* em = getenv("CFLX_LOOKAHEAD_MULTI");  // multi-rank grids: on by default (validated on 2x2x1 / 1x1x2)
        const bool want = (e ? atoi(e) != 0 : true) && (lu->P == 1 || !em || atoi(em) != 0);
        if (want) {
            CFLX_TRY(handle_side_stream(lu.get()));
            CFLX_TRY(lu->ev_fork.create(cudaEventDisableTiming));
            CFLX_TRY(lu->ev_join.create(cudaEventDisableTiming));
            const char* c = getenv("CFLX_PANEL_CTAS");
            // SMs of the look-ahead pivot search: fewer on one GPU (no tournament), more where the tournament exchanges
            // sit on the critical path; CFLX_PANEL_CTAS overrides
            lu->pws.cta_cap = c ? atoi(c) : (lu->P == 1 ? 32 : (lu->Px == 1 ? 48 : 64));
        }
    }
    // zero the panels once: padded columns are read (and masked) by the GEMM producer
    cudaMemsetAsync(lu->PT, 0, pan * sizeof(double), c->stream);
    cudaMemsetAsync(lu->PT2, 0, pan * sizeof(double), c->stream);
    cudaMemsetAsync(lu->LT, 0, pan * sizeof(double), c->stream);
    cudaMemsetAsync(lu->W, 0, pan * sizeof(double), c->stream);
    cudaMemsetAsync(lu->A01raw, 0, upan * sizeof(double), c->stream);
    cudaMemsetAsync(lu->U, 0, upan * sizeof(double), c->stream);
    cudaMemsetAsync(lu->A0, 0, (size_t)lu->Ml * lu->Nl * sizeof(double), c->stream);
    CFLX_CUDA(cudaStreamSynchronize(c->stream));
    *out = lu.release();
    return CFLX_OK;
}

int cflx_lu_info(const cflx_lu* lu, int* o) {
    REFUSE_IF(!lu);
    REFUSE_IF(!o);
    const int vals[16] = {lu->M, lu->N, lu->Ml, lu->Nl, lu->Nt, lu->nlayr, lu->P, lu->Px, lu->Py, lu->Pz, lu->pi, lu->pj,
                          lu->pk, lu->rank, lu->v, 0};
    std::memcpy(o, vals, sizeof(vals));
    return CFLX_OK;
}

int cflx_lu_set_local(cflx_lu* lu, const double* host_local) {
    REFUSE_IF(!lu);
    REFUSE_IF(!host_local);
    CFLX_TRY(enter(lu, __func__, 0));
    CFLX_TRY(handle_set_local(lu, host_local));
    lu->rbt.in.depth = 0;
    lu->next_host = nullptr;
    return CFLX_OK;
}

// Input streaming for back-to-back factorisations: the NEXT cflx_lu_factor call uploads `host_next` (page-locked memory,
// valid until that call returns) into the input buffer on a copy stream as soon as it has taken its own working copy of
// the current input, so the 8*Ml*Nl-byte transfer overlaps the factorisation; the factorisation after that consumes it
// without a cflx_lu_set_local.  The residual of a run whose input buffer was handed to the next matrix is refused.
int cflx_lu_queue_next_local(cflx_lu* lu, const double* host_next) {
    REFUSE_IF(!lu);
    REFUSE_IF(!host_next);
    CFLX_TRY(enter(lu, __func__, NEED_INPUT));
    if (!lu->copy) {
        CFLX_TRY(lu->copy.create(cudaStreamNonBlocking));
        CFLX_TRY(lu->ev_a0_read.create(cudaEventDisableTiming));
        CFLX_TRY(lu->ev_upload.create(cudaEventDisableTiming));
    }
    lu->next_host = host_next;
    return CFLX_OK;
}

}  // extern "C"

namespace {
// The factorisation both entry points share, from the working copy of the input to the timeline: the pivot search of
// cflx_lu_factor, or with lu->fixed the prescribed order of cflx_lu_factor_fixed (fixed_panel).  COLLECTIVE.
int lu_factor_run(cflx_lu* lu, double* ms_out) {
    cflx_comm* c = lu->comm;
    cudaStream_t s = c->stream;
    const size_t loc = (size_t)lu->Ml * lu->Nl;
    lu->perm_done = false;
    // "init" region of the reference (conflux_opt.hpp:347-515): A11Buff = copy of gv.data, gri, counters
    {
        PhaseTimer t(lu, RG_init, s);
        if (lu->a0_is_next) CFLX_CUDA(cudaStreamWaitEvent(s, lu->ev_upload, 0));  // this run's input was streamed in
        CFLX_CUDA(cudaMemcpyAsync(lu->A11, lu->A0, loc * sizeof(double), cudaMemcpyDeviceToDevice, s));
    }
    lu->a0_is_next = false;
    lu->sv.ready = false;
    // the factors carry the input's scaling and transform; a queued next input arrives unscaled and untransformed
    CFLX_TRY(equil_pass_on(&lu->eq, lu->M, lu->next_host != nullptr, s));
    CFLX_TRY(rbt_pass_on(&lu->rbt, lu->M, lu->next_host != nullptr, s));
    if (lu->next_host) {  // queued next input: overwrite A0 behind the working copy, concurrently with everything below
        CFLX_CUDA(cudaEventRecord(lu->ev_a0_read, s));
        CFLX_CUDA(cudaStreamWaitEvent(lu->copy, lu->ev_a0_read, 0));
        CFLX_CUDA(cudaMemcpyAsync(lu->A0, lu->next_host, loc * sizeof(double), cudaMemcpyHostToDevice, lu->copy));
        CFLX_CUDA(cudaEventRecord(lu->ev_upload, lu->copy));
        lu->next_host = nullptr;
        lu->a0_is_next = true;
    }
    CFLX_TRY(launch_iota_gri(lu->gri, lu->igri, lu->Ml, lu->v, lu->Px, lu->pi, s));
    for (double& x : lu->phase_ms) x = 0;
    for (int sd = 0; sd < 2; ++sd)
        for (int r = 0; r < RG_COUNT; ++r) lu->region_ms[sd][r] = 0, lu->region_cnt[sd][r] = 0;
    lu->tl_recs.clear();
    lu->tl_spans.clear();
    CFLX_TRY(grid_barrier(c));  // MPI_Barrier(lu_comm) before t1 (conflux_opt.hpp:531)
    Events<2> loop;
    CFLX_TRY(loop.create());
    CFLX_CUDA(cudaEventRecord(loop[0], s));
    int fnpr = 0;
    lu->gemm_flops = 0;
    lu->gemm_ms = 0;
    if (lu->time_gemm && (int)lu->ev.size() < 4 * lu->Nt) {
        lu->ev = std::vector<Event>(4 * lu->Nt);
        for (Event& e : lu->ev) CFLX_TRY(e.create());
    }
    lu->ev_used.assign(2 * lu->Nt, 0);
    {
        cudaStream_t side = (lu->prof_mode == 1) ? nullptr : lu->side.s;
        if (side) {
            CFLX_CUDA(cudaEventRecord(lu->ev_fork, s));
            CFLX_CUDA(cudaStreamWaitEvent(side, lu->ev_fork, 0));
        }
        CFLX_TRY(panel_phase(lu, 0, 0, side ? side : s));
        if (side) {
            CFLX_CUDA(cudaEventRecord(lu->ev_join, side));
            CFLX_CUDA(cudaStreamWaitEvent(s, lu->ev_join, 0));
        }
    }
    for (int k = 0; k < lu->Nt; ++k) CFLX_TRY(finish_step(lu, k, fnpr));
    CFLX_CUDA(cudaEventRecord(loop[1], s));
    CFLX_CUDA(cudaEventSynchronize(loop[1]));
    float ms = 0;
    CFLX_CUDA(cudaEventElapsedTime(&ms, loop[0], loop[1]));
    CFLX_CUDA(cudaGetLastError());
    if (ms_out) *ms_out = ms;
    if (lu->prof_mode == 2) {  // resolve the timeline: every event has completed (e1 was synchronised, the side stream joined)
        if (lu->side) cudaStreamSynchronize(lu->side);
        for (const auto& r : lu->tl_recs) {
            float g = 0;
            if (cudaEventElapsedTime(&g, lu->tl_pool[r.ev], lu->tl_pool[r.ev + 1]) == cudaSuccess) {
                lu->region_ms[r.side][r.region] += g;
                lu->region_cnt[r.side][r.region]++;
                lu->phase_ms[region_phase(r.region)] += g;
                float st = 0;
                if (cudaEventElapsedTime(&st, lu->tl_pool[0], lu->tl_pool[r.ev]) != cudaSuccess) cudaGetLastError();
                lu->tl_spans.push_back({r.region, r.side, st, g});
            } else {
                cudaGetLastError();
            }
        }
    }
    if (lu->time_gemm) {
        for (int i = 0; i < 2 * lu->Nt; ++i) {
            if (!lu->ev_used[i]) continue;
            float g = 0;
            if (cudaEventElapsedTime(&g, lu->ev[2 * i], lu->ev[2 * i + 1]) == cudaSuccess) lu->gemm_ms += g;
            else cudaGetLastError();
        }
    }
    if (lu->a0_is_next) CFLX_CUDA(cudaStreamSynchronize(lu->copy));  // the caller's staging buffer is free again
    lu->factored = true;
    lu->low_prec = lu->update.tf32();
    lu->perm_done = true;
    return CFLX_OK;
}

// FNV-1a over the words of the order: what the ranks compare before a fixed factorisation
unsigned long long order_hash(const std::vector<int>& p) {
    unsigned long long h = 1469598103934665603ull;
    for (int x : p) {
        h ^= (unsigned)x;
        h *= 1099511628211ull;
    }
    return h;
}

}  // namespace

// min(~w) = ~max(w)
int cflx::world_agree(Handle* lu, bool ok, std::initializer_list<unsigned long long> words, bool* same) {
    cflx_comm* c = lu->comm;
    if (c->world_size == 1) {
        *same = ok;
        return CFLX_OK;
    }
    const size_t n = words.size();
    std::vector<unsigned long long> w(words);
    for (unsigned long long x : words) w.push_back(~x);
    w.push_back(ok ? 1ull : 0ull);
    CFLX_TRY(lu->agree.grow(w.size()));
    CFLX_CUDA(cudaMemcpyAsync(lu->agree, w.data(), sizeof(w[0]) * w.size(), cudaMemcpyHostToDevice, c->stream));
    CFLX_NCCL(ncclAllReduce(lu->agree, lu->agree, w.size(), ncclUint64, ncclMin, c->world, c->stream));
    CFLX_CUDA(cudaMemcpyAsync(w.data(), lu->agree, sizeof(w[0]) * w.size(), cudaMemcpyDeviceToHost, c->stream));
    CFLX_CUDA(cudaStreamSynchronize(c->stream));
    *same = w[2 * n] == 1;
    for (size_t i = 0; i < n; ++i) *same = *same && w[i] == ~w[n + i];
    return CFLX_OK;
}

namespace {

// The checks of cflx_lu_factor_fixed (`who`) that need no other rank; on success lu->fix_perm_h holds the order and the
// device buffers of the fixed path exist
int fixed_prepare(const char* who, cflx_lu* lu, const int* perm, double tiny, const int* info_out) {
    REFUSE_FOR(who, !(tiny >= 0.0));
    REFUSE_FOR(who, !info_out);
    CFLX_TRY(enter(lu, who, NEED_INPUT));
    const int M = lu->M;
    std::vector<int>& p = lu->fix_perm_h;
    if (perm) {
        p.assign(perm, perm + M);
    } else {
        if (!lu->perm_done) {
            set_last_error("%s: perm = NULL before any factorisation of this handle completed", who);
            return CFLX_ERR_STATE;
        }
        // the permutation of the last factorisation, which set_local keeps
        CFLX_TRY(lu_permutation(lu, &p));
    }
    std::vector<char> seen(M, 0);
    for (int x : p) {
        if (x < 0 || x >= M || seen[x]) {
            set_last_error("%s: perm is not a permutation of [0, %d)", who, M);
            return CFLX_ERR_ARG;
        }
        seen[x] = 1;
    }
    if (!lu->fix_perm) CFLX_TRY(lu->fix_perm.alloc(M));
    if (!lu->fix_rec) CFLX_TRY(lu->fix_rec.alloc(4));
    const size_t ws = getrf_nopiv_scratch(lu->v, getrf_nopiv_blocked(lu->v));
    if (ws && !lu->fix_ws) CFLX_TRY(lu->fix_ws.alloc(ws));
    return CFLX_OK;
}

// The checks of cflx_lu_rbt (`who`) that need no other rank
int rbt_prepare(const char* who, cflx_lu* lu, int depth) {
    REFUSE_FOR(who, depth < 1);
    REFUSE_FOR(who, depth > 4);
    if (lu->rbt.in.depth) {
        set_last_error("%s: refused, the input is already transformed; upload it again first", who);
        return CFLX_ERR_STATE;
    }
    CFLX_TRY(enter(lu, who, NEED_INPUT | NEED_UNSCALED));
    const long long q = (long long)lu->v * lu->Px << depth;
    if (lu->M % q) {
        set_last_error("%s: M = %d is not a multiple of 2^%d v Px = %lld; the smallest M that works is %lld: "
                       "pad A with the identity to that order", who, lu->M, depth, q, (lu->M + q - 1) / q * q);
        return CFLX_ERR_UNSUPPORTED;
    }
    return CFLX_OK;
}

}  // namespace

extern "C" {

int cflx_lu_factor(cflx_lu* lu, double* ms_out) {
    REFUSE_IF(!lu);
    CFLX_TRY(enter(lu, __func__, NEED_INPUT));
    return lu_factor_run(lu, ms_out);
}

// COLLECTIVE.  P A = L U with the P of a prescribed order: the arguments agreed on by every rank first (one world
// all-reduce, so that a refusal anywhere is a refusal everywhere and no rank enters the loop alone), then the shared
// factorisation with fixed_panel in place of the pivot search, then the replacements (sum) and the first zero pivot (min)
// combined over the world.
int cflx_lu_factor_fixed(cflx_lu* lu, const int* perm, double tiny, int* nrepl_out, int* info_out, double* ms_out) {
    REFUSE_IF(!lu);
    CFLX_TRY(enter(lu, __func__, 0));  // the device of world_agree, whatever fixed_prepare finds
    cflx_comm* c = lu->comm;
    cudaStream_t s = c->stream;
    const int rc = fixed_prepare(__func__, lu, perm, tiny, info_out);
    bool same = false;
    CFLX_TRY(world_agree(lu, rc == CFLX_OK, {rc == CFLX_OK ? order_hash(lu->fix_perm_h) : 0}, &same));
    if (rc != CFLX_OK) return rc;
    if (!same) {
        set_last_error("%s: the ranks passed different orders, or another rank refused its arguments", __func__);
        return CFLX_ERR_ARG;
    }
    const int v = lu->v, Px = lu->Px;
    const std::vector<int>& p = lu->fix_perm_h;
    lu->fix_npiv.assign(lu->Nt, 0);
    for (int q = 0; q < lu->Nt * v; ++q)
        if ((p[q] / v) % Px == lu->pi) lu->fix_npiv[q / v]++;
    CFLX_CUDA(cudaMemcpyAsync(lu->fix_perm, p.data(), sizeof(int) * lu->M, cudaMemcpyHostToDevice, s));
    CFLX_CUDA(cudaMemsetAsync(lu->fix_rec, 0, 4 * sizeof(int), s));
    lu->fix_tiny = tiny;
    lu->fixed = true;
    const int run = lu_factor_run(lu, ms_out);
    lu->fixed = false;
    CFLX_TRY(run);
    CFLX_TRY(launch_fixed_info_operand(lu->fix_rec, s));
    lu->launches++;
    if (c->world_size > 1) {
        CFLX_NCCL(ncclGroupStart());
        CFLX_NCCL(ncclAllReduce(lu->fix_rec, lu->fix_rec, 1, ncclInt, ncclSum, c->world, s));
        CFLX_NCCL(ncclAllReduce(lu->fix_rec + 2, lu->fix_rec + 2, 1, ncclInt, ncclMin, c->world, s));
        CFLX_NCCL(ncclGroupEnd());
    }
    int rec[4] = {0, 0, 0, 0};
    CFLX_CUDA(cudaMemcpyAsync(rec, lu->fix_rec, sizeof(rec), cudaMemcpyDeviceToHost, s));
    CFLX_CUDA(cudaStreamSynchronize(s));
    if (nrepl_out) *nrepl_out = rec[0];
    *info_out = rec[2] == INT_MAX ? 0 : rec[2];
    return CFLX_OK;
}

// COLLECTIVE.  A0 <- U^T A0 V on every rank's share (rbt.cu), after the ranks agreed on depth and seed with one world
// all-reduce, so that a refusal anywhere is a refusal everywhere.  The input changes: the factors and the solve cache
// are dropped, as by an equilibration that scales the input.
int cflx_lu_rbt(cflx_lu* lu, int depth, uint64_t seed, double* u_out, double* v_out) {
    REFUSE_IF(!lu);
    CFLX_TRY(enter(lu, __func__, 0));  // the device of world_agree, whatever rbt_prepare finds
    const int rc = rbt_prepare(__func__, lu, depth);
    bool same = false;
    CFLX_TRY(world_agree(lu, rc == CFLX_OK, {seed, (unsigned long long)depth}, &same));
    if (rc != CFLX_OK) return rc;
    if (!same) {
        set_last_error("%s: the ranks passed different depths or seeds, or another rank refused its arguments", __func__);
        return CFLX_ERR_ARG;
    }
    const int M = lu->M;
    const size_t n = (size_t)depth * M;
    std::vector<double> r(2 * n), sc(2 * n);
    rbt_multipliers(M, depth, seed, 0, r.data());
    rbt_multipliers(M, depth, seed, 1, r.data() + n);
    if (u_out) std::memcpy(u_out, r.data(), sizeof(double) * n);
    if (v_out) std::memcpy(v_out, r.data() + n, sizeof(double) * n);
    rbt_scales(r.data(), 2 * n, sc.data());
    cudaStream_t s = lu->comm->stream;
    if (lu->a0_is_next) CFLX_CUDA(cudaStreamWaitEvent(s, lu->ev_upload, 0));  // A0 holds a streamed next input
    lu->factored = false;
    lu->sv.ready = false;
    RbtRecord& in = lu->rbt.in;
    CFLX_TRY(rbt_record_set(&in, depth, seed, sc.data(), M, s));
    if (lu->pk == 0) CFLX_TRY(launch_rbt(RbtOp::W, lu->A0, lu->Nl, *lu, lu->Nl, INT_MAX, depth, in.s, in.s + n, s));
    CFLX_CUDA(cudaStreamSynchronize(s));  // sc is a host temporary
    return CFLX_OK;
}

// COLLECTIVE.  op(A) X = B through the transformed system the factors represent: B to the device, U^T (V^T) on its rows,
// the solve with W (W^T), dgerfs on that system with refine, V (U) on the rows of X; svx_tail with the butterflies as its
// row transforms.
int cflx_lu_rbt_solve(cflx_lu* lu, int trans, int nrhs, const double* B, int ldb, double* X, int ldx, int refine,
                      double* ferr_out, double* berr_out) {
    REFUSE_IF(!lu);
    REFUSE_IF(trans != 0 && trans != 1);
    REFUSE_IF(refine != 0 && refine != 1);
    CFLX_TRY(rhs_args(__func__, nrhs, B, ldb, X, ldx, true));
    CFLX_TRY(enter(lu, __func__, NEED_FACTORS | NEED_FP64 | (refine ? NEED_OWN_INPUT : 0u)));
    if (!lu->rbt.fac.depth) {
        set_last_error("%s: the factors carry no random butterfly transform (cflx_lu_rbt before the factorisation)",
                       __func__);
        return CFLX_ERR_STATE;
    }
    const bool t = trans != 0;
    const RefineOp op = lu_refine_op(lu, t);
    auto refine_step = [&](const double* dB, int lb, double* dX, int lx) {
        return refine ? refine_run(&lu->sv.rf, op, nrhs, dB, lb, dX, lx, ferr_out, berr_out) : CFLX_OK;
    };
    return svx_tail(&lu->eq, op, nrhs, B, ldb, X, ldx, rbt_rows(*lu, t ? RbtOp::VT : RbtOp::UT),
                    rbt_rows(*lu, t ? RbtOp::U : RbtOp::V), refine_step);
}

// Not collective.  One of the factors' butterflies on the rows of this rank's right-hand side share (rbt.cu); a host
// share goes through one temporary device share.
int cflx_lu_rbt_apply_local(cflx_lu* lu, int op, int nrhs, double* B_local, int ldb) {
    REFUSE_IF(!lu);
    REFUSE_IF(op < 0);
    REFUSE_IF(op > 3);
    REFUSE_IF(nrhs < 1);
    REFUSE_IF(!B_local);
    const int ncl = rhs_local_cols(nrhs, lu->v, lu->Py);
    REFUSE_IF(ldb < ncl);
    return rbt_apply_local(__func__, "cflx_lu_rbt", lu, (RbtOp)op, nrhs, B_local, ldb);
}

int cflx_lu_get_permutation(cflx_lu* lu, int* perm_out) {
    REFUSE_IF(!lu);
    REFUSE_IF(!perm_out);
    CFLX_TRY(enter(lu, __func__, NEED_FACTORS));
    std::vector<int> hist;
    CFLX_TRY(lu_permutation(lu, &hist));
    std::memcpy(perm_out, hist.data(), sizeof(int) * lu->M);
    return CFLX_OK;
}

// Rows of the finished factors live where their original row lives (local rows are in the order they were
// promoted).  The reference's validation layout wants pivoted row q = k*v + i on rank (k % Px, pj, 0) at local
// row (k / Px)*v + i (conflux_opt.hpp:1673-1699,1721-1754): an all-to-all of whole rows inside each grid column.
int cflx_lu_get_factors(cflx_lu* lu, double* C_host, int* perm_out) {
    REFUSE_IF(!lu);
    CFLX_TRY(enter(lu, __func__, NEED_FACTORS));
    cudaStream_t s = lu->comm->stream;
    std::vector<int> hist;
    CFLX_TRY(lu_permutation(lu, &hist));
    if (perm_out) std::memcpy(perm_out, hist.data(), sizeof(int) * lu->M);
    if (lu->pk != 0) return CFLX_OK;  // only layer 0 holds factors
    const size_t loc = (size_t)lu->Ml * lu->Nl;
    if (!lu->Cbuf) CFLX_TRY(lu->Cbuf.alloc(loc));
    CFLX_TRY(redistribute_pivoted_rows(lu, hist, true, lu->A11, lu->Cbuf));
    if (C_host) CFLX_CUDA(cudaMemcpyAsync(C_host, lu->Cbuf, loc * sizeof(double), cudaMemcpyDeviceToHost, s));
    CFLX_CUDA(cudaStreamSynchronize(s));
    return CFLX_OK;
}

// ||P A - L U||_F (absolute, what the reference's validation build prints, conflux_miniapp.cpp:494-500) and the same
// relative to ||A||_F, computed on the device grid with the library's own GEMM + NCCL (validate.cu).  COLLECTIVE.
int cflx_lu_validate(cflx_lu* lu, double* frob_abs_out, double* frob_rel_out) {
    REFUSE_IF(!lu);
    return lu_validate(__func__, lu, frob_abs_out, frob_rel_out);
}
int cflx_lu_residual(cflx_lu* lu, double* rel_out) {
    REFUSE_IF(!lu);
    REFUSE_IF(!rel_out);
    return lu_validate(__func__, lu, nullptr, rel_out);
}

// Reads only the factors, so a run whose input buffer was handed to the queued next matrix can still be solved.
int cflx_lu_solve(cflx_lu* lu, int nrhs, const double* B, int ldb, double* X, int ldx) {
    REFUSE_IF(!lu);
    CFLX_TRY(rhs_args(__func__, nrhs, B, ldb, X, ldx, false));
    CFLX_TRY(enter(lu, __func__, NEED_FACTORS | NEED_FP64));
    return lu_sweeps(lu, false, false, nrhs, B, ldb, X, ldx);
}

// A^T X = B with the same factors and state rules: U^T Y = B, L^T W = Y by column-partial sweeps, then X = P^T W.
int cflx_lu_solve_trans(cflx_lu* lu, int nrhs, const double* B, int ldb, double* X, int ldx) {
    REFUSE_IF(!lu);
    CFLX_TRY(rhs_args(__func__, nrhs, B, ldb, X, ldx, false));
    CFLX_TRY(enter(lu, __func__, NEED_FACTORS | NEED_FP64));
    return lu_sweeps(lu, true, false, nrhs, B, ldb, X, ldx);
}

// COLLECTIVE.  A X = B or A^T X = B with B and X distributed like A (solve_local.cu): each block of columns assembled on
// the device and solved by the sweeps of cflx_lu_solve / cflx_lu_solve_trans, then scattered into X's share.
int cflx_lu_solve_local(cflx_lu* lu, int trans, int nrhs, const double* B_local, int ldb, double* X_local, int ldx) {
    REFUSE_IF(!lu);
    REFUSE_IF(trans != 0 && trans != 1);
    SolveLocalArgs a{};
    CFLX_TRY(solve_local_args(__func__, *lu, nrhs, B_local, ldb, X_local, ldx, &a));
    CFLX_TRY(enter(lu, __func__, NEED_FACTORS | NEED_FP64));
    auto solve = [lu, trans](int, int w, double* Bk, double*, int ldn, const double** Xk) -> int {
        CFLX_TRY(lu_sweeps(lu, trans != 0, false, w, Bk, ldn, nullptr, 0));
        *Xk = trans ? lu->sv.Xg : lu->sv.X;  // the transposed solve's P^T lands in Xg
        return CFLX_OK;
    };
    return solve_local_run(*lu, solve_local_rows(*lu, false), a, inverse_block_cols(lu->M, lu->v), false, solve);
}

// LAPACK dgecon (NORM = '1') on the grid (lu_rcond).
int cflx_lu_rcond(cflx_lu* lu, double* rcond_out, double* anorm_out) {
    REFUSE_IF(!lu);
    REFUSE_IF(!rcond_out);
    CFLX_TRY(enter(lu, __func__, NEED_FACTORS | NEED_FP64 | NEED_OWN_INPUT));
    return lu_rcond(lu, false, rcond_out, anorm_out);
}

// COLLECTIVE.  LAPACK dgetri on the grid (inverse.cu): the first exactly zero U(k,k) over the world, then the block
// solves with the identity, each block column q of inv(P A) landing in column perm[q] of this rank's share.  Reads only
// the factors and the permutation, like cflx_lu_solve.
int cflx_lu_inverse(cflx_lu* lu, double* Ainv_local, int* info_out) {
    REFUSE_IF(!lu);
    REFUSE_IF(!info_out);
    CFLX_TRY(enter(lu, __func__, NEED_FACTORS | NEED_FP64));
    if (!lu->sv.ready) CFLX_TRY(lu_solve_prepare(lu));
    int info = 0;
    CFLX_TRY(zero_pivot_grid(*lu, &lu->eq, lu->Cbuf, &info));
    *info_out = info;
    if (info > 0) return CFLX_OK;  // exactly singular U: no inverse, nothing written
    return inverse_run(&lu->sv, lu_solve_factor(lu), InvKind::LU, lu->hist, Ainv_local);
}

// COLLECTIVE.  det(A) = det(P) det(U) (det.cu): the diagonal of U from Cbuf, its exact-range product, divided by the
// products of the scales when unscaled; det(P) from the cycles of the permutation, the same on every rank.
int cflx_lu_det(cflx_lu* lu, int unscaled, double* sign_out, double* logabsdet_out, double* mant_out, int64_t* exp_out,
                int* info_out) {
    REFUSE_IF(!lu);
    REFUSE_IF(unscaled != 0 && unscaled != 1);
    REFUSE_IF(!info_out);
    CFLX_TRY(enter(lu, __func__, NEED_FACTORS | NEED_FP64));
    if (!lu->sv.ready) CFLX_TRY(lu_solve_prepare(lu));
    const EquilRecord& eq = lu->eq.fac;
    const double* r = unscaled && (eq.equed == 'R' || eq.equed == 'B') ? eq.r.p : nullptr;
    const double* c = unscaled && (eq.equed == 'C' || eq.equed == 'B') ? eq.c.p : nullptr;
    DetResult d{};
    CFLX_TRY(det_grid(*lu, &lu->eq, lu->Cbuf, false, r, c, &d));
    std::vector<int> perm;
    CFLX_TRY(lu_permutation(lu, &perm));
    // det(P) = (-1)^(M - number of cycles): a cycle of length L is L - 1 transpositions
    std::vector<char> seen(lu->M, 0);
    int odd = d.neg;
    for (int i = 0; i < lu->M; ++i)
        for (int j = i; !seen[j]; j = perm[j]) {
            seen[j] = 1;
            odd ^= j != i;
        }
    const double sign = d.nonfinite ? std::nan("") : d.first_zero ? 0.0 : odd ? -1.0 : 1.0;
    if (sign_out) *sign_out = sign;
    if (logabsdet_out) *logabsdet_out = det_log(d);
    if (mant_out) *mant_out = d.mant;
    if (exp_out) *exp_out = d.exp;
    *info_out = d.first_zero;
    return CFLX_OK;
}

// COLLECTIVE.  LAPACK dgerfs on the grid: residuals of the input A0 (refine.cu), corrections and the forward-error
// estimator's products by the solves above (lu_refine_op).
int cflx_lu_refine(cflx_lu* lu, int trans, int nrhs, const double* B, int ldb, double* X, int ldx, double* ferr_out,
                   double* berr_out) {
    REFUSE_IF(!lu);
    REFUSE_IF(trans != 0 && trans != 1);
    CFLX_TRY(rhs_args(__func__, nrhs, B, ldb, X, ldx, true));
    CFLX_TRY(enter(lu, __func__, NEED_FACTORS | NEED_FP64 | NEED_OWN_INPUT));
    return refine_run(&lu->sv.rf, lu_refine_op(lu, trans != 0), nrhs, B, ldb, X, ldx, ferr_out, berr_out);
}

// COLLECTIVE.  LAPACK dgerfsx on the grid: the first exactly zero U(k,k), dgecon of A0 in the infinity-norm (trans 0) or
// the 1-norm (trans 1), then refine_x_run with the scales of the solution's rows: c for trans 0 (equed C / B), r for
// trans 1 (equed R / B).
int cflx_lu_refine_x(cflx_lu* lu, int trans, int nrhs, const double* B, int ldb, double* X, int ldx, double* rcond_out,
                     double* berr_out, double* err_bnds_norm_out, double* err_bnds_comp_out, int* info_out) {
    REFUSE_IF(!lu);
    REFUSE_IF(trans != 0 && trans != 1);
    CFLX_TRY(rhs_args(__func__, nrhs, B, ldb, X, ldx, true));
    REFUSE_IF(!err_bnds_norm_out);
    REFUSE_IF(!info_out);
    CFLX_TRY(enter(lu, __func__, NEED_FACTORS | NEED_FP64 | NEED_OWN_INPUT));
    const bool t = trans != 0;
    double rcond = 0.0;
    int info = 0;
    CFLX_TRY(lu_expert_pre(lu, !t, nullptr, false, &rcond, &info));
    *info_out = info;
    if (rcond_out) *rcond_out = rcond;
    if (info > 0) return CFLX_OK;  // exactly singular U: X is left as it was
    return refine_x_run(&lu->sv.rf, lu_refine_op(lu, t), nrhs, B, ldb, X, ldx, lu_scales(lu, t).post, rcond,
                        err_bnds_comp_out != nullptr, berr_out, err_bnds_norm_out, err_bnds_comp_out, info_out);
}

// COLLECTIVE.  LAPACK dgeequ (+ dlaqge when apply) on the input A0 (equil.cu).  The input changes, so the factorisation
// and the solve cache are dropped, as by cflx_lu_set_local.
int cflx_lu_equilibrate(cflx_lu* lu, int apply, double* r_out, double* c_out, double* rowcnd_out, double* colcnd_out,
                        double* amax_out, char* equed_out, int* info_out) {
    return lu_equilibrate(__func__, lu, apply, false, r_out, c_out, rowcnd_out, colcnd_out, amax_out, equed_out, info_out);
}

// COLLECTIVE.  LAPACK dgeequb (+ dlaqge when apply): cflx_lu_equilibrate with the scales rounded to powers of two.
int cflx_lu_equilibrate_b(cflx_lu* lu, int apply, double* r_out, double* c_out, double* rowcnd_out, double* colcnd_out,
                          double* amax_out, char* equed_out, int* info_out) {
    return lu_equilibrate(__func__, lu, apply, true, r_out, c_out, rowcnd_out, colcnd_out, amax_out, equed_out, info_out);
}

// COLLECTIVE.  LAPACK dgesvxx after the factorisation, with the scaling the factors carry: the first zero pivot and
// dla_gerpvgrw, then B scaled, the solve, dgerfsx's refinement as cflx_lu_refine_x runs it, X unscaled.
int cflx_lu_svxx(cflx_lu* lu, int trans, int nrhs, const double* B, int ldb, double* X, int ldx, double* rcond_out,
                 double* rpvgrw_out, double* berr_out, double* err_bnds_norm_out, double* err_bnds_comp_out,
                 char* equed_out, int* info_out) {
    REFUSE_IF(!lu);
    REFUSE_IF(trans != 0 && trans != 1);
    CFLX_TRY(rhs_args(__func__, nrhs, B, ldb, X, ldx, true));
    REFUSE_IF(!rcond_out);
    REFUSE_IF(!err_bnds_norm_out);
    REFUSE_IF(!info_out);
    CFLX_TRY(enter(lu, __func__, NEED_FACTORS | NEED_FP64 | NEED_OWN_INPUT));
    const bool t = trans != 0;
    if (equed_out) *equed_out = lu->eq.fac.equed;
    double rpvgrw = 1.0, rcond = 0.0;
    int info = 0;
    // dgecon as cflx_lu_refine_x: the infinity-norm for trans 0, the 1-norm for trans 1
    CFLX_TRY(lu_expert_pre(lu, !t, &rpvgrw, true, &rcond, &info));
    if (rpvgrw_out) *rpvgrw_out = rpvgrw;
    *info_out = info;
    *rcond_out = rcond;
    if (info > 0) return CFLX_OK;  // exactly singular U: X is left as it was
    // B is scaled by the scales of the rows of op(A), X (and the bounds' d) by those of its columns
    const LuScales sc = lu_scales(lu, t);
    return svxx_run(&lu->eq, &lu->sv.rf, lu_refine_op(lu, t), nrhs, B, ldb, X, ldx, sc.pre, sc.post, sc.post, rcond,
                    err_bnds_comp_out != nullptr, berr_out, err_bnds_norm_out, err_bnds_comp_out, info_out);
}

// COLLECTIVE.  LAPACK dgesvx after the factorisation, with the scaling the factors carry: B scaled, the reciprocal pivot
// growth and the first zero pivot, rcond (1-norm for trans 0, infinity-norm for trans 1), the solve, dgerfs, X unscaled.
int cflx_lu_svx(cflx_lu* lu, int trans, int nrhs, const double* B, int ldb, double* X, int ldx, double* rcond_out,
                double* ferr_out, double* berr_out, double* rpvgrw_out, char* equed_out, int* info_out) {
    REFUSE_IF(!lu);
    REFUSE_IF(trans != 0 && trans != 1);
    CFLX_TRY(rhs_args(__func__, nrhs, B, ldb, X, ldx, true));
    REFUSE_IF(!rcond_out);
    REFUSE_IF(!info_out);
    CFLX_TRY(enter(lu, __func__, NEED_FACTORS | NEED_FP64 | NEED_OWN_INPUT));
    const bool t = trans != 0;
    if (equed_out) *equed_out = lu->eq.fac.equed;
    double rpvgrw = 1.0, rcond = 0.0;
    int info = 0;
    // dgecon with NORM = '1' (trans 0, as cflx_lu_rcond) or 'I' (trans 1)
    CFLX_TRY(lu_expert_pre(lu, t, &rpvgrw, false, &rcond, &info));
    if (rpvgrw_out) *rpvgrw_out = rpvgrw;
    *info_out = info;
    *rcond_out = rcond;
    if (info > 0) return CFLX_OK;  // exactly singular U: no solution
    // op(A) X = B: B is scaled by the scales of the rows of op(A), X by those of its columns
    const LuScales sc = lu_scales(lu, t);
    return svx_run(&lu->eq, &lu->sv.rf, lu_refine_op(lu, t), nrhs, B, ldb, X, ldx, ferr_out, berr_out, sc.pre, sc.post,
                   sc.cnd, rcond, info_out);
}

// ---------------------------------------------------------------- refinement and the expert drivers, B and X distributed
// Each block of refine_block_cols columns is assembled as cflx_lu_solve_local assembles it (with X for refine and
// refine_x), run through the replicated driver's core on device buffers, and scattered; the matrix-level parts run once
// before the loop.  So each block's bits are those of the replicated driver called on those columns alone.

// COLLECTIVE.  cflx_lu_refine with B and X distributed like A.
int cflx_lu_refine_local(cflx_lu* lu, int trans, int nrhs, const double* B_local, int ldb, double* X_local, int ldx,
                         double* ferr_out, double* berr_out) {
    REFUSE_IF(!lu);
    REFUSE_IF(trans != 0 && trans != 1);
    SolveLocalArgs a{};
    CFLX_TRY(refine_local_args(__func__, *lu, nrhs, B_local, ldb, X_local, ldx, true, &a));
    CFLX_TRY(enter(lu, __func__, NEED_FACTORS | NEED_FP64 | NEED_OWN_INPUT));
    const RefineOp op = lu_refine_op(lu, trans != 0);
    auto run = [&](int c0, int w, double* Bk, double* Xk, int ldn, const double** out) -> int {
        *out = Xk;
        return refine_run(&lu->sv.rf, op, w, Bk, ldn, Xk, ldn, ferr_out ? ferr_out + c0 : nullptr,
                          berr_out ? berr_out + c0 : nullptr);
    };
    return solve_local_run(*lu, solve_local_rows(*lu, false), a, refine_block_cols(lu->v), true, run);
}

// COLLECTIVE.  cflx_lu_refine_x with B and X distributed like A: the zero-pivot check and dgecon once, then the blocks.
int cflx_lu_refine_x_local(cflx_lu* lu, int trans, int nrhs, const double* B_local, int ldb, double* X_local, int ldx,
                           double* rcond_out, double* berr_out, double* err_bnds_norm_out, double* err_bnds_comp_out,
                           int* info_out) {
    REFUSE_IF(!lu);
    REFUSE_IF(trans != 0 && trans != 1);
    SolveLocalArgs a{};
    CFLX_TRY(refine_local_args(__func__, *lu, nrhs, B_local, ldb, X_local, ldx, true, &a));
    REFUSE_IF(!err_bnds_norm_out);
    REFUSE_IF(!info_out);
    CFLX_TRY(enter(lu, __func__, NEED_FACTORS | NEED_FP64 | NEED_OWN_INPUT));
    const bool t = trans != 0;
    double rcond = 0.0;
    int info = 0;
    CFLX_TRY(lu_expert_pre(lu, !t, nullptr, false, &rcond, &info));
    *info_out = info;
    if (rcond_out) *rcond_out = rcond;
    if (info > 0) return CFLX_OK;  // exactly singular U: X is left as it was
    const RefineOp op = lu_refine_op(lu, t);
    const double* d = lu_scales(lu, t).post;
    auto run = [&](int c0, int w, double* Bk, double* Xk, int ldn, const double** out) -> int {
        *out = Xk;
        int bi = 0;
        CFLX_TRY(refine_x_run(&lu->sv.rf, op, w, Bk, ldn, Xk, ldn, d, rcond, err_bnds_comp_out != nullptr,
                              berr_out ? berr_out + c0 : nullptr, err_bnds_norm_out + 3 * (size_t)c0,
                              err_bnds_comp_out ? err_bnds_comp_out + 3 * (size_t)c0 : nullptr, &bi));
        merge_block_info(&info, bi, c0);
        return CFLX_OK;
    };
    CFLX_TRY(solve_local_run(*lu, solve_local_rows(*lu, false), a, refine_block_cols(lu->v), true, run));
    *info_out = info;
    return CFLX_OK;
}

// COLLECTIVE.  cflx_lu_svx with B and X distributed like A: the pivot growth, the zero-pivot check and dgecon once,
// then the blocks; X output only.
int cflx_lu_svx_local(cflx_lu* lu, int trans, int nrhs, const double* B_local, int ldb, double* X_local, int ldx,
                      double* rcond_out, double* ferr_out, double* berr_out, double* rpvgrw_out, char* equed_out,
                      int* info_out) {
    REFUSE_IF(!lu);
    REFUSE_IF(trans != 0 && trans != 1);
    SolveLocalArgs a{};
    CFLX_TRY(refine_local_args(__func__, *lu, nrhs, B_local, ldb, X_local, ldx, false, &a));
    REFUSE_IF(!rcond_out);
    REFUSE_IF(!info_out);
    CFLX_TRY(enter(lu, __func__, NEED_FACTORS | NEED_FP64 | NEED_OWN_INPUT));
    const bool t = trans != 0;
    if (equed_out) *equed_out = lu->eq.fac.equed;
    double rpvgrw = 1.0, rcond = 0.0;
    int info = 0;
    CFLX_TRY(lu_expert_pre(lu, t, &rpvgrw, false, &rcond, &info));
    if (rpvgrw_out) *rpvgrw_out = rpvgrw;
    *info_out = info;
    *rcond_out = rcond;
    if (info > 0) return CFLX_OK;  // exactly singular U: X is not written
    const RefineOp op = lu_refine_op(lu, t);
    const LuScales sc = lu_scales(lu, t);
    auto run = [&](int c0, int w, double* Bk, double*, int ldn, const double** out) -> int {
        *out = Bk;  // svx_tail reads B before it writes X
        return svx_run(&lu->eq, &lu->sv.rf, op, w, Bk, ldn, Bk, ldn, ferr_out ? ferr_out + c0 : nullptr,
                       berr_out ? berr_out + c0 : nullptr, sc.pre, sc.post, sc.cnd, rcond, info_out);
    };
    return solve_local_run(*lu, solve_local_rows(*lu, false), a, refine_block_cols(lu->v), false, run);
}

// COLLECTIVE.  cflx_lu_svxx with B and X distributed like A: dla_gerpvgrw, the zero-pivot check and dgecon once, then
// the blocks; X output only.
int cflx_lu_svxx_local(cflx_lu* lu, int trans, int nrhs, const double* B_local, int ldb, double* X_local, int ldx,
                       double* rcond_out, double* rpvgrw_out, double* berr_out, double* err_bnds_norm_out,
                       double* err_bnds_comp_out, char* equed_out, int* info_out) {
    REFUSE_IF(!lu);
    REFUSE_IF(trans != 0 && trans != 1);
    SolveLocalArgs a{};
    CFLX_TRY(refine_local_args(__func__, *lu, nrhs, B_local, ldb, X_local, ldx, false, &a));
    REFUSE_IF(!rcond_out);
    REFUSE_IF(!err_bnds_norm_out);
    REFUSE_IF(!info_out);
    CFLX_TRY(enter(lu, __func__, NEED_FACTORS | NEED_FP64 | NEED_OWN_INPUT));
    const bool t = trans != 0;
    if (equed_out) *equed_out = lu->eq.fac.equed;
    double rpvgrw = 1.0, rcond = 0.0;
    int info = 0;
    CFLX_TRY(lu_expert_pre(lu, !t, &rpvgrw, true, &rcond, &info));
    if (rpvgrw_out) *rpvgrw_out = rpvgrw;
    *info_out = info;
    *rcond_out = rcond;
    if (info > 0) return CFLX_OK;  // exactly singular U: X is not written
    const RefineOp op = lu_refine_op(lu, t);
    const LuScales sc = lu_scales(lu, t);
    auto run = [&](int c0, int w, double* Bk, double*, int ldn, const double** out) -> int {
        *out = Bk;
        int bi = 0;
        CFLX_TRY(svxx_run(&lu->eq, &lu->sv.rf, op, w, Bk, ldn, Bk, ldn, sc.pre, sc.post, sc.post, rcond,
                          err_bnds_comp_out != nullptr, berr_out ? berr_out + c0 : nullptr,
                          err_bnds_norm_out + 3 * (size_t)c0, err_bnds_comp_out ? err_bnds_comp_out + 3 * (size_t)c0 : nullptr,
                          &bi));
        merge_block_info(&info, bi, c0);
        return CFLX_OK;
    };
    CFLX_TRY(solve_local_run(*lu, solve_local_rows(*lu, false), a, refine_block_cols(lu->v), false, run));
    *info_out = info;
    return CFLX_OK;
}

// COLLECTIVE.  LAPACK dsgesv on the grid: the input factored with the TF32 trailing update (prec 1: one term, 3: three),
// a zero pivot of that U checked over the world, then mixed_run's refinement in FP64 on A0.  When the low-precision
// factors fail (iter -3) or the loop does not converge (-31), the input is factored again in FP64 and solved, as
// cflx_lu_factor + cflx_lu_solve do; the handle then holds those FP64 factors.
int cflx_lu_sv_mixed(cflx_lu* lu, int prec, int nrhs, const double* B, int ldb, double* X, int ldx, int itmax,
                     int* iter_out, double* berr_out, double* ms_out) {
    REFUSE_IF(!lu);
    REFUSE_IF(prec != CFLX_PREC_TF32 && prec != CFLX_PREC_TF32X3);
    REFUSE_IF(!iter_out);
    CFLX_TRY(rhs_args(__func__, nrhs, B, ldb, X, ldx, true));
    CFLX_TRY(enter(lu, __func__, NEED_INPUT | NEED_UNSCALED));
    if (lu->rbt.in.depth) {
        set_last_error("%s: refused, the input carries a random butterfly transform (cflx_lu_rbt); upload it again first",
                       __func__);
        return CFLX_ERR_STATE;
    }
    if (lu->next_host) {
        set_last_error("%s: refused, a next input is queued (cflx_lu_queue_next_local): the refinement reads this input "
                       "after the factorisation", __func__);
        return CFLX_ERR_STATE;
    }
    double ms = 0.0;
    CFLX_TRY(lu->update.with_tf32(prec, [&] { return lu_factor_run(lu, &ms); }));
    double anorm = 0.0;
    CFLX_TRY(norminf_grid(*lu, lu->A0, &anorm));
    CFLX_TRY(lu_solve_prepare(lu));
    int zero = 0, iter = MIXED_LOW_PREC_FAILED;
    CFLX_TRY(zero_pivot_grid(*lu, &lu->eq, lu->Cbuf, &zero));
    if (zero == 0)
        CFLX_TRY(mixed_run(&lu->sv.rf, lu_refine_op(lu, false), anorm, itmax > 0 ? itmax : MIXED_ITMAX, nrhs, B, ldb, X,
                           ldx, &iter, berr_out));
    if (iter < 0) {
        double ms2 = 0.0;
        CFLX_TRY(lu_factor_run(lu, &ms2));
        ms += ms2;
        CFLX_TRY(lu_sweeps(lu, false, false, nrhs, B, ldb, X, ldx));
        if (berr_out) CFLX_TRY(mixed_berr(&lu->sv.rf, lu_refine_op(lu, false), anorm, nrhs, B, ldb, X, ldx, berr_out));
    }
    *iter_out = iter;
    if (ms_out) *ms_out = ms;
    return CFLX_OK;
}

int cflx_host_alloc(size_t bytes, void** out) {
    REFUSE_IF(!out);
    if (device_count() == 0) {
        set_last_error("%s: no CUDA device visible: conflux_b200 has no CPU fallback", __func__);
        return CFLX_ERR_NO_DEVICE;
    }
    CFLX_CUDA(cudaHostAlloc(out, bytes, cudaHostAllocPortable));
    return CFLX_OK;
}
int cflx_host_free(void* p) {
    if (p) CFLX_CUDA(cudaFreeHost(p));
    return CFLX_OK;
}

int cflx_lu_uses_ozaki(const cflx_lu* lu) { return lu && lu->update.int8 ? 1 : 0; }
int cflx_lu_launch_count(cflx_lu* lu, int64_t* count_out, int reset) {
    REFUSE_IF(!lu);
    REFUSE_IF(!count_out);
    return handle_launch_count(lu, count_out, reset);
}
int cflx_lu_set_profiling(cflx_lu* lu, int mode) {  // 0 off, 1 serialising phase timers, 2 non-serialising timeline
    REFUSE_IF(!lu);
    REFUSE_IF(mode < 0);
    REFUSE_IF(mode > 2);
    lu->prof_mode = mode;
    return CFLX_OK;
}
// JSON text {"main": {region: [ms, count], ...}, "side": {...}, "records": [[region, "main" | "side", start ms, ms], ...]}
// of the last profiled cflx_lu_factor; region names are the reference's semiprof regions.  "records" (profiling mode 2
// only) lists every region instance in launch order, start relative to the first recorded event.  Returns the length
// needed (incl. the terminator) when buf is too small.
int cflx_lu_timeline(cflx_lu* lu, char* buf, int buf_len) {
    REFUSE_IF(!lu);
    std::string o = "{";
    for (int sd = 0; sd < 2; ++sd) {
        o += sd ? ", \"side\": {" : "\"main\": {";
        bool first = true;
        for (int r = 0; r < RG_COUNT; ++r) {
            if (!lu->region_cnt[sd][r]) continue;
            char tmp[160];
            snprintf(tmp, sizeof(tmp), "%s\"%s\": [%.4f, %d]", first ? "" : ", ", region_name(r), lu->region_ms[sd][r], lu->region_cnt[sd][r]);
            o += tmp;
            first = false;
        }
        o += "}";
    }
    o += ", \"records\": [";
    for (size_t i = 0; i < lu->tl_spans.size(); ++i) {
        const auto& sp = lu->tl_spans[i];
        char tmp[160];
        snprintf(tmp, sizeof(tmp), "%s[\"%s\", \"%s\", %.4f, %.4f]", i ? ", " : "", region_name(sp.region), sp.side ? "side" : "main",
                 sp.start_ms, sp.ms);
        o += tmp;
    }
    o += "]}";
    if (!buf || buf_len <= (int)o.size()) return (int)o.size() + 1;
    std::memcpy(buf, o.c_str(), o.size() + 1);
    return CFLX_OK;
}
int cflx_lu_phase_ms(cflx_lu* lu, double* ms_out) {
    REFUSE_IF(!lu);
    REFUSE_IF(!ms_out);
    for (int i = 0; i < PH_COUNT; ++i) ms_out[i] = lu->phase_ms[i];
    return CFLX_OK;
}
int cflx_lu_set_kernel_timing(cflx_lu* lu, int enabled) {
    REFUSE_IF(!lu);
    lu->time_gemm = enabled != 0;
    return CFLX_OK;
}
int cflx_lu_trailing_stats(cflx_lu* lu, double* ms_out, double* flops_out) {
    REFUSE_IF(!lu);
    REFUSE_IF(!ms_out);
    REFUSE_IF(!flops_out);
    *ms_out = lu->gemm_ms;
    *flops_out = lu->gemm_flops;
    return CFLX_OK;
}
void cflx_lu_destroy(cflx_lu* lu) { delete lu; }

}  // extern "C"

cflx_lu::~cflx_lu() {
    cudaSetDevice(comm->device);
    for (SubComm* sc : {&jk_comm, &ik_comm})
        if (sc->c) ncclCommDestroy(sc->c);
    grid_free(this);
}
