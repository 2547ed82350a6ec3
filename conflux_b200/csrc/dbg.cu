// conflux_b200/csrc/dbg.cu -- single-device test / micro-benchmark hooks of the C ABI (cflx_dbg_*).
// They drive the SAME kernels the factorisation uses, with host buffers in and out, so that tests/ can check every
// kernel in isolation against numpy / the oracle, and bench.py can time the dominant kernel alone.
#include <algorithm>
#include <climits>
#include <limits>
#include <vector>

#include "../../include/conflux_b200.h"
#include "common.cuh"
#include "kernels.h"
#include "lu_state.h"

using namespace cflx;

namespace {
int check_device() {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) {
        cudaGetLastError();
        set_last_error("no CUDA device visible: conflux_b200 has no CPU fallback");
        return CFLX_ERR_NO_DEVICE;
    }
    return CFLX_OK;
}

// the conditions on a cflx_share_layout that differ between hooks (see the header)
enum : unsigned { TILED = 1, COVERED = 2, NONEMPTY = 4 };

// *L = the share *s describes, or the refusal of hook `who` naming the first condition it fails: those of every share,
// then those `need` adds
int share_layout(const char* who, const cflx_share_layout* s, unsigned need, Layout* L) {
    if (!s) return refuse(who, "no share layout");
    const auto [M, v, Kappa, Ml, Nl, Px, Py, pi, pj] = *s;
    if (v < 1) return refuse(who, "v < 1");
    if (Px < 1 || Py < 1) return refuse(who, "Px or Py < 1");
    if (pi < 0 || pi >= Px) return refuse(who, "pi outside [0, Px)");
    if (pj < 0 || pj >= Py) return refuse(who, "pj outside [0, Py)");
    if (Ml < 0 || Nl < 0) return refuse(who, "Ml or Nl < 0");
    if ((need & NONEMPTY) && (Ml < 1 || Nl < 1)) return refuse(who, "Ml or Nl < 1");
    if ((need & TILED) && (Ml % v || Nl % v)) return refuse(who, "Ml or Nl not a multiple of v");
    if ((need & COVERED) && (M < (Ml / v) * Px * v || M < (Nl / v) * Py * v))
        return refuse(who, "M < (Ml / v) Px v or M < (Nl / v) Py v");
    *L = Layout{M, v, Kappa, Ml, Nl, Px, Py, pi, pj};
    return CFLX_OK;
}

// d = a device buffer of n T (with DevBuf's tail pad) holding the host array h, or uninitialised when h is null
template <class T = double>
int stage(DevBuf<>& d, size_t n, const T* h = nullptr) {
    CFLX_TRY(d.alloc(sizeof(T) * n));
    if (h) CFLX_CUDA(cudaMemcpy(d.p, h, sizeof(T) * n, cudaMemcpyHostToDevice));
    return CFLX_OK;
}
// h = the first n T of the device array d, when h is not null
template <class T>
int fetch(T* h, const void* d, size_t n) {
    if (h) CFLX_CUDA(cudaMemcpy(h, d, sizeof(T) * n, cudaMemcpyDeviceToHost));
    return CFLX_OK;
}

// *ms_out (may be null) = the mean device time of `reps` (at least 1) back-to-back calls of run() on the default
// stream, after one warm-up call
template <class Run>
int time_reps(Run&& run, int reps, double* ms_out) {
    Events<2> ev;
    CFLX_TRY(ev.create());
    if (reps < 1) reps = 1;
    CFLX_TRY(run());  // warm-up
    CFLX_CUDA(cudaEventRecord(ev[0]));
    for (int r = 0; r < reps; ++r) CFLX_TRY(run());
    CFLX_CUDA(cudaEventRecord(ev[1]));
    CFLX_CUDA(cudaEventSynchronize(ev[1]));
    float ms = 0;
    CFLX_CUDA(cudaEventElapsedTime(&ms, ev[0], ev[1]));
    if (ms_out) *ms_out = ms / reps;
    return CFLX_OK;
}

// a residual kernel (refine.cu) on the share A of layout L: launch(mode, A, Xc, Xr, P, Q) runs it on the device copies
// of A, Xc (Nl x nrhs) and Xr (Ml x nrhs).  The timed repetitions run first, then the launch whose result is returned,
// into zeroed outputs of rows x nrhs (Ml, Nl or Ml + Nl rows by mode).
template <class Launch>
int residual_run(int mode, const Layout& L, const double* A, int nrhs, const double* Xc, const double* Xr, double* P_out,
                 double* Q_out, int reps, double* ms_out, Launch&& launch) {
    const ResidMode m = mode == 0 ? ResidMode::NN : mode == 1 ? ResidMode::TN : ResidMode::SymLower;
    const int rows = mode == 0 ? L.Ml : mode == 1 ? L.Nl : L.Ml + L.Nl;
    const size_t o_n = (size_t)std::max(rows, 1) * nrhs;
    DevBuf<> dA, dXc, dXr, dP, dQ;
    CFLX_TRY(stage(dA, (size_t)L.Ml * L.Nl, A));
    CFLX_TRY(stage(dXc, (size_t)L.Nl * nrhs, Xc));
    CFLX_TRY(stage(dXr, (size_t)L.Ml * nrhs, Xr));
    CFLX_TRY(stage(dP, o_n));
    CFLX_TRY(stage(dQ, o_n));
    double *p = dP.as<double>(), *q = dQ.as<double>();
    auto run = [&] { return launch(m, dA.as<double>(), dXc.as<double>(), dXr.as<double>(), p, q); };
    CFLX_TRY(time_reps(run, reps, ms_out));
    CFLX_CUDA(cudaMemset(dP.p, 0, sizeof(double) * o_n));
    CFLX_CUDA(cudaMemset(dQ.p, 0, sizeof(double) * o_n));
    CFLX_TRY(run());
    CFLX_TRY(fetch(P_out, dP.p, (size_t)rows * nrhs));
    CFLX_TRY(fetch(Q_out, dQ.p, (size_t)rows * nrhs));
    CFLX_CUDA(cudaDeviceSynchronize());
    return CFLX_OK;
}

// one of the solve's narrow GEMMs on staged operands: launch(C, D) runs it on the device copy of C (M x N, c_n entries;
// null: zeros).  The timed repetitions write a separate output; the result is one more launch on the pristine inputs,
// into C itself when D == C (the kernel with D aliasing C).
template <class Launch>
int narrow_gemm(size_t c_n, const double* C, double* D, int reps, double* ms_out, Launch&& launch) {
    DevBuf<> dC, dT;
    CFLX_TRY(stage(dC, c_n, C));
    CFLX_TRY(stage(dT, c_n));
    if (!C) CFLX_CUDA(cudaMemset(dC.p, 0, sizeof(double) * c_n));
    CFLX_TRY(time_reps([&] { return launch(dC.as<double>(), dT.as<double>()); }, reps, ms_out));
    double* out = C && D == C ? dC.as<double>() : dT.as<double>();
    CFLX_TRY(launch(dC.as<double>(), out));
    CFLX_TRY(fetch(D, out, c_n));
    CFLX_CUDA(cudaDeviceSynchronize());
    return CFLX_OK;
}

// ---- FP64 pipe peak probes ------------------------------------------------------------------------------
__global__ void dmma_peak_kernel(double* out, int iters) {
    double c[16][2];
#pragma unroll
    for (int i = 0; i < 16; ++i) c[i][0] = c[i][1] = 0.0;
    double a = 1.0 + threadIdx.x * 1e-9, b = 1.0 - threadIdx.x * 1e-9;
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int i = 0; i < 16; ++i) dmma884(c[i][0], c[i][1], a, b);
    }
    double s = 0;
#pragma unroll
    for (int i = 0; i < 16; ++i) s += c[i][0] + c[i][1];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
// m16n8kK, K = 4, 8, 16: 16 independent accumulator chains per warp, so the probe measures issue rate, not latency
template <int K>
__global__ void dmma16x8_peak_kernel(double* out, int iters) {
    double c[16][4];
#pragma unroll
    for (int i = 0; i < 16; ++i) c[i][0] = c[i][1] = c[i][2] = c[i][3] = 0.0;
    double a[K / 2], b[K / 4];
#pragma unroll
    for (int i = 0; i < K / 2; ++i) a[i] = 1.0 + (threadIdx.x + i) * 1e-9;
#pragma unroll
    for (int i = 0; i < K / 4; ++i) b[i] = 1.0 - (threadIdx.x + i) * 1e-9;
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            if constexpr (K == 4) dmma16x8x4(c[i], a, b[0]);
            else if constexpr (K == 8) dmma16x8x8(c[i], a, b);
            else dmma16x8x16(c[i], a, b);
        }
    }
    double s = 0;
#pragma unroll
    for (int i = 0; i < 16; ++i) s += c[i][0] + c[i][1] + c[i][2] + c[i][3];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
__global__ void dfma_peak_kernel(double* out, int iters) {
    double c[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) c[i] = i;
    double a = 1.0 + threadIdx.x * 1e-9, b = 1e-9;
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int i = 0; i < 16; ++i) c[i] = fma(c[i], a, b);
    }
    double s = 0;
#pragma unroll
    for (int i = 0; i < 16; ++i) s += c[i];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
}  // namespace

extern "C" {

// which: 0 = the shape gemm_tn_kernel issues (m16n8k8), 1 = DFMA, 2/3/4 = mma m16n8k4/k8/k16 f64, 5 = mma m8n8k4 f64.
// burst = best of a few short launches (what a kernel timed alone can reach at the maximum clock); sustained = one
// launch 256x longer (what survives the power cap inside a long step)
int cflx_dbg_fp64_peak_ex(int which, double* burst_out, double* sustained_out) {
    CFLX_TRY(check_device());
    if (which == 0) which = 3;
    if (which < 1 || which > 5) {
        set_last_error("fp64_peak: unknown probe %d", which);
        return CFLX_ERR_ARG;
    }
    int dev = 0, sms = 0;
    CFLX_CUDA(cudaGetDevice(&dev));
    CFLX_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const int threads = 256, blocks = sms * 4;
    DevBuf<> out;
    CFLX_TRY(out.alloc(sizeof(double) * threads * blocks));
    Events<2> ev;
    CFLX_TRY(ev.create());
    // flop per warp instruction: m16n8kK = 2*16*8*K (1024 / 2048 / 4096), m8n8k4 = 512; DFMA = 2 flop per lane.
    // The larger shapes run proportionally fewer iterations, so every probe's launches do about the same work.
    const double per_warp_instr = which == 2 ? 1024.0 : which == 3 ? 2048.0 : which == 4 ? 4096.0 : 512.0;
    const int shrink = which == 1 ? 1 : (int)(per_warp_instr / 512.0);
    auto run = [&](int iters, double* tf) -> int {
        iters /= shrink;
        CFLX_CUDA(cudaEventRecord(ev[0]));
        switch (which) {
            case 1: dfma_peak_kernel<<<blocks, threads>>>(out.as<double>(), iters); break;
            case 2: dmma16x8_peak_kernel<4><<<blocks, threads>>>(out.as<double>(), iters); break;
            case 3: dmma16x8_peak_kernel<8><<<blocks, threads>>>(out.as<double>(), iters); break;
            case 4: dmma16x8_peak_kernel<16><<<blocks, threads>>>(out.as<double>(), iters); break;
            default: dmma_peak_kernel<<<blocks, threads>>>(out.as<double>(), iters); break;
        }
        CFLX_CUDA(cudaGetLastError());
        CFLX_CUDA(cudaEventRecord(ev[1]));
        CFLX_CUDA(cudaEventSynchronize(ev[1]));
        float ms = 0;
        CFLX_CUDA(cudaEventElapsedTime(&ms, ev[0], ev[1]));
        const double flop = which == 1 ? (double)blocks * threads * iters * 16 * 2.0
                                       : (double)blocks * (threads / 32) * iters * 16 * per_warp_instr;
        *tf = flop / (ms * 1e-3) / 1e12;
        return CFLX_OK;
    };
    double burst = 0, tf = 0;
    for (int rep = 0; rep < 4; ++rep) {
        CFLX_TRY(run(1024, &tf));
        if (rep > 0 && tf > burst) burst = tf;
    }
    double sustained = 0;
    CFLX_TRY(run(262144, &sustained));
    if (burst_out) *burst_out = burst;
    if (sustained_out) *sustained_out = sustained;
    return CFLX_OK;
}
int cflx_dbg_fp64_peak(int which, double* tflops_out) { return cflx_dbg_fp64_peak_ex(which, tflops_out, nullptr); }

// gemm_tn_kernel on a window of whole buffers, as the factorisation and the TRSMs launch it (see the header).  The
// timed repetitions run first; then C (and D) are restored and the launch whose result is returned runs.
int cflx_dbg_gemm_tn(int M, int N, int K, const double* AT, int at_rows, int64_t ldat, int64_t at_off, const double* B,
                     int b_rows, int64_t ldb, int64_t b_off, const double* C, int c_rows, int64_t ldc, int row_off,
                     int col_off, double alpha, double beta, int in_place, double* D_out, double* C_out, int reps,
                     double* ms_out) {
    CFLX_TRY(check_device());
    REFUSE_IF(M <= 0 || N <= 0 || K <= 0);
    REFUSE_IF(!AT || !B || !C);
    REFUSE_IF(at_rows <= 0 || b_rows <= 0 || c_rows <= 0 || ldat <= 0 || ldb <= 0 || ldc <= 0);
    REFUSE_IF(at_off < 0 || b_off < 0 || row_off < 0 || col_off < 0);
    // every element the kernel may touch lies inside the buffers: AT rows of round_up(M, 2) (the producer's even copy
    // width), B rows of N, the C window; 16-byte alignment of every operand row needs even offsets
    if ((at_off & 1) || (b_off & 1) || (col_off & 1) || at_off + (K - 1) * ldat + round_up(M, 2) > (int64_t)at_rows * ldat ||
        b_off + (K - 1) * ldb + N > (int64_t)b_rows * ldb || row_off + M > c_rows || col_off + N > ldc)
        return refuse(__func__, "window outside the buffers or misaligned");
    const size_t a_n = (size_t)at_rows * ldat, b_n = (size_t)b_rows * ldb, c_n = (size_t)c_rows * ldc;
    DevBuf<> dA, dB, dC, dC0, dD;
    CFLX_TRY(stage(dA, a_n, AT));
    CFLX_TRY(stage(dB, b_n, B));
    CFLX_TRY(stage(dC, c_n));
    CFLX_TRY(stage(dC0, c_n, C));
    CFLX_TRY(stage(dD, c_n));
    auto restore = [&]() -> int {
        CFLX_CUDA(cudaMemcpy(dC.p, dC0.p, sizeof(double) * c_n, cudaMemcpyDeviceToDevice));
        CFLX_CUDA(cudaMemcpy(dD.p, dC0.p, sizeof(double) * c_n, cudaMemcpyDeviceToDevice));
        return CFLX_OK;
    };
    const int64_t c_at = (int64_t)row_off * ldc + col_off;
    GemmArgs g{};
    g.M = M; g.N = N; g.K = K;
    g.AT = dA.as<double>() + at_off; g.ldat = ldat;
    g.B = dB.as<double>() + b_off; g.ldb = ldb;
    g.C = dC.as<double>() + c_at; g.ldc = ldc;
    g.D = (in_place ? dC.as<double>() : dD.as<double>()) + c_at; g.ldd = ldc;
    g.alpha = alpha; g.beta = beta;
    CFLX_TRY(restore());
    CFLX_TRY(time_reps([&] { return launch_gemm_tn(g, 0); }, reps, ms_out));
    CFLX_TRY(restore());
    CFLX_TRY(launch_gemm_tn(g, 0));
    CFLX_TRY(fetch(D_out, in_place ? dC.p : dD.p, c_n));
    CFLX_TRY(fetch(C_out, dC.p, c_n));
    CFLX_CUDA(cudaDeviceSynchronize());
    return CFLX_OK;
}

// D = beta*C + alpha * A * B on the narrow GEMM of the solve (solve.cu); A [M x K], B [K x N], C / D [M x N] dense
// row-major.  D == C (the same host array) runs the kernel with D aliasing C on the device.
int cflx_dbg_gemm_narrow(int M, int N, int K, const double* A, const double* B, const double* C, double alpha, double beta,
                         double* D, int reps, double* ms_out) {
    CFLX_TRY(check_device());
    REFUSE_IF(M <= 0 || N <= 0 || K < 0);
    REFUSE_IF(K & 3);
    REFUSE_IF(!A || !B);
    DevBuf<> dA, dB;
    CFLX_TRY(stage(dA, (size_t)M * K, A));
    CFLX_TRY(stage(dB, (size_t)K * N, B));
    return narrow_gemm((size_t)M * N, C, D, reps, ms_out, [&](const double* c, double* out) {
        return launch_gemm_narrow(M, N, K, dA.as<double>(), K, dB.as<double>(), N, c, N, out, N, alpha, beta, 0);
    });
}

// D = beta*C + alpha * AT^T * B on the transposed narrow GEMM (solve.cu), like cflx_dbg_gemm_narrow; AT [K x M] is stored
// on the device with the even leading dimension round_up(M, 2), the kernel's condition, so odd M can be run.
int cflx_dbg_gemm_narrow_tn(int M, int N, int K, const double* AT, const double* B, const double* C, double alpha,
                            double beta, double* D, int reps, double* ms_out) {
    CFLX_TRY(check_device());
    REFUSE_IF(M <= 0 || N <= 0 || K < 0);
    REFUSE_IF(!AT || !B);
    const int64_t ldat = round_up(M, 2);
    DevBuf<> dA, dB;
    CFLX_TRY(stage(dA, K * ldat));
    CFLX_TRY(stage(dB, (size_t)K * N, B));
    if (K > 0) CFLX_CUDA(cudaMemcpy2D(dA.p, ldat * 8, AT, (size_t)M * 8, (size_t)M * 8, K, cudaMemcpyHostToDevice));
    return narrow_gemm((size_t)M * N, C, D, reps, ms_out, [&](const double* c, double* out) {
        return launch_gemm_narrow_tn(M, N, K, dA.as<double>(), ldat, dB.as<double>(), N, c, N, out, N, alpha, beta, 0);
    });
}

// the narrow GEMM (trans: the transposed one) on a window of whole buffers, as the solve engine launches it (see the
// header)
int cflx_dbg_gemm_narrow_window(int trans, int M, int N, int K, const double* A, int a_rows, int64_t lda, int a_row,
                                int a_col, const double* B, int b_rows, int64_t ldb, int b_row, int b_col, const double* C,
                                int c_rows, int64_t ldc, int c_row, int c_col, double alpha, double beta, int in_place,
                                double* D_out, double* C_out) {
    CFLX_TRY(check_device());
    const char* who = __func__;
    if (M < 1 || N < 1 || K < 0) return refuse(who, "M < 1, N < 1 or K < 0");
    if (!A || !B || !C) return refuse(who, "A, B or C is null");
    if (a_rows < 1 || b_rows < 1 || c_rows < 1 || lda < 1 || ldb < 1 || ldc < 1)
        return refuse(who, "a buffer with no rows or a leading dimension < 1");
    if (a_row < 0 || a_col < 0 || b_row < 0 || b_col < 0 || c_row < 0 || c_col < 0) return refuse(who, "negative offset");
    if (!trans && (K & 3)) return refuse(who, "K not a multiple of 4");
    if ((lda & 1) || (a_col & 1)) return refuse(who, "odd lda or A column offset (A rows must be 16-byte aligned)");
    // the A block: M rows of K (trans: K rows of M); B: K rows of N; the C window: M rows of N
    const int a_h = trans ? K : M, a_w = trans ? M : K;
    if ((int64_t)a_row + a_h > a_rows || a_col + (int64_t)a_w > lda) return refuse(who, "A block outside its buffer");
    if ((int64_t)b_row + K > b_rows || b_col + (int64_t)N > ldb) return refuse(who, "B block outside its buffer");
    if ((int64_t)c_row + M > c_rows || c_col + (int64_t)N > ldc) return refuse(who, "C window outside its buffer");
    const size_t a_n = (size_t)a_rows * lda, b_n = (size_t)b_rows * ldb, c_n = (size_t)c_rows * ldc;
    DevBuf<> dA, dB, dC, dD;
    CFLX_TRY(stage(dA, a_n, A));
    CFLX_TRY(stage(dB, b_n, B));
    CFLX_TRY(stage(dC, c_n, C));
    CFLX_TRY(stage(dD, c_n, C));
    const double* a = dA.as<double>() + (int64_t)a_row * lda + a_col;
    const double* b = dB.as<double>() + (int64_t)b_row * ldb + b_col;
    const int64_t c_at = (int64_t)c_row * ldc + c_col;
    double* c = dC.as<double>() + c_at;
    double* d = (in_place ? dC.as<double>() : dD.as<double>()) + c_at;
    if (trans)
        CFLX_TRY(launch_gemm_narrow_tn(M, N, K, a, lda, b, ldb, c, ldc, d, ldc, alpha, beta, 0));
    else
        CFLX_TRY(launch_gemm_narrow(M, N, K, a, lda, b, ldb, c, ldc, d, ldc, alpha, beta, 0));
    CFLX_TRY(fetch(D_out, in_place ? dC.p : dD.p, c_n));
    CFLX_TRY(fetch(C_out, dC.p, c_n));
    CFLX_CUDA(cudaDeviceSynchronize());
    return CFLX_OK;
}

// one diagonal tile of the solve engine: its inverse blocks as solve_inverses makes them, then diag_solve (see the header)
int cflx_dbg_diag_solve(int tri, int lower, int v, int nb, const double* share, int rows, int64_t ld, int row0, int col0,
                        int ldn, const double* R, double* Y_out, double* inv_out) {
    CFLX_TRY(check_device());
    const char* who = __func__;
    if (tri < 0 || tri > 4) return refuse(who, "tri outside 0 .. 4");
    if (lower != 0 && lower != 1) return refuse(who, "lower not 0 or 1");
    const Tri t = static_cast<Tri>(tri);
    if (lower ? (t != Tri::Lower && t != Tri::LowerT) : t == Tri::LowerT)
        return refuse(who, "tri not one the solves use on this kind of tile");
    if (nb != 4 && nb != 8 && nb != 16 && nb != 32 && nb != 64 && nb != 128)
        return refuse(who, "nb not 4, 8, 16, 32, 64 or 128", CFLX_ERR_UNSUPPORTED);
    if (v < nb || v % nb) return refuse(who, "v not a positive multiple of nb");
    if (ldn < 1) return refuse(who, "ldn < 1");
    if (!share || !R || !Y_out) return refuse(who, "share, R or Y_out is null");
    if (row0 < 0 || col0 < 0) return refuse(who, "negative tile offset");
    if ((ld & 1) || (col0 & 1)) return refuse(who, "odd ld or col0 (the tile's rows must be 16-byte aligned)");
    if ((int64_t)row0 + v > rows || col0 + (int64_t)v > ld) return refuse(who, "tile outside the share");
    const size_t blocks = 2 * (size_t)v * nb, rn = (size_t)v * ldn;
    DevBuf<> dS, dInv, dTile, dLinvT, dR, dY;
    CFLX_TRY(stage(dS, (size_t)rows * ld, share));
    CFLX_TRY(stage(dInv, blocks));
    CFLX_TRY(stage(dTile, (size_t)v * v));
    CFLX_TRY(stage(dLinvT, (size_t)v * nb));
    CFLX_TRY(stage(dR, rn, R));
    CFLX_TRY(stage(dY, rn));
    const double* ftt = dS.as<double>() + (int64_t)row0 * ld + col0;
    CFLX_TRY(solve_tile_inverses(ftt, ld, v, nb, lower != 0, dInv.as<double>(), dTile.as<double>(), dLinvT.as<double>(), 0));
    CFLX_TRY(diag_solve(dInv.as<double>(), ftt, ld, v, nb, t, dR.as<double>(), dY.as<double>(), ldn, 0));
    CFLX_TRY(fetch(Y_out, dY.p, rn));
    CFLX_TRY(fetch(inv_out, dInv.p, blocks));
    CFLX_CUDA(cudaDeviceSynchronize());
    return CFLX_OK;
}

// the per-share kernels of equilibration and of the pivot growth (equil.cu) on one layer-0 share; each output may be null
int cflx_dbg_equil(const cflx_share_layout* share, const double* A, const double* r, const double* c, char equed, int ncols,
                   double* rowmax_out, double* colmax_out, double* diag_out, double* scaled_out, double* sym_scaled_out,
                   double* growth_out, int* zero_pivot_out) {
    CFLX_TRY(check_device());
    Layout L;
    CFLX_TRY(share_layout(__func__, share, TILED | COVERED, &L));
    REFUSE_IF(!A || !r || !c);
    REFUSE_IF(equed != 'N' && equed != 'R' && equed != 'C' && equed != 'B');
    const int M = L.M;
    const size_t a_n = (size_t)L.Ml * L.Nl;
    DevBuf<> dA, dW, dr, dc, dv, dg, dz;
    CFLX_TRY(stage(dA, a_n, A));
    CFLX_TRY(stage(dW, a_n));
    CFLX_TRY(stage(dr, M, r));
    CFLX_TRY(stage(dc, M, c));
    CFLX_TRY(stage(dv, M));
    CFLX_TRY(stage(dg, 2 * (size_t)M));
    CFLX_TRY(stage<int>(dz, 1));
    const double* a = dA.as<double>();
    double *w = dW.as<double>(), *vec = dv.as<double>();
    if (rowmax_out) CFLX_TRY(equil_row_max(a, L, vec, 0));
    CFLX_TRY(fetch(rowmax_out, vec, M));
    if (colmax_out) CFLX_TRY(equil_col_max(a, L, dr.as<double>(), vec, 0));
    CFLX_TRY(fetch(colmax_out, vec, M));
    if (diag_out) CFLX_TRY(equil_diag(a, L, vec, 0));
    CFLX_TRY(fetch(diag_out, vec, M));
    if (scaled_out) {
        CFLX_CUDA(cudaMemcpy(w, a, sizeof(double) * a_n, cudaMemcpyDeviceToDevice));
        CFLX_TRY(equil_apply(w, L, dr.as<double>(), dc.as<double>(), equed, 0));
        CFLX_TRY(fetch(scaled_out, w, a_n));
    }
    if (sym_scaled_out) {  // s = r
        CFLX_CUDA(cudaMemcpy(w, a, sizeof(double) * a_n, cudaMemcpyDeviceToDevice));
        CFLX_TRY(equil_sym_apply(w, L, dr.as<double>(), 0));
        CFLX_TRY(fetch(sym_scaled_out, w, a_n));
    }
    if (growth_out) {  // the share is both L\U and the input; dgesvx's maxima are those of the columns' maxima
        CFLX_TRY(equil_growth_cols(a, a, L, false, ncols, dg.as<double>(), 0));
        std::vector<double> h(2 * (size_t)M);
        CFLX_TRY(fetch(h.data(), dg.p, h.size()));
        growth_out[0] = *std::max_element(h.begin() + M, h.end());
        growth_out[1] = *std::max_element(h.begin(), h.begin() + M);
    }
    if (zero_pivot_out) {
        CFLX_TRY(equil_zero_pivot(a, L, dz.as<int>(), 0));
        int z = 0;
        CFLX_TRY(fetch(&z, dz.p, 1));
        *zero_pivot_out = z == INT_MAX ? 0 : z;
    }
    CFLX_CUDA(cudaDeviceSynchronize());
    return CFLX_OK;
}

// the per-column pivot growth pass (equil.cu) on one layer-0 share F (the factor) and A (the input); mode 0 LU, 1
// Cholesky; either output may be null
int cflx_dbg_growth_cols(int mode, const cflx_share_layout* share, int ncols, const double* F, const double* A,
                         double* amax_out, double* fmax_out) {
    CFLX_TRY(check_device());
    Layout L;
    CFLX_TRY(share_layout(__func__, share, TILED | COVERED, &L));
    REFUSE_IF(mode != 0 && mode != 1);
    REFUSE_IF(!F || !A);
    const size_t a_n = (size_t)L.Ml * L.Nl;
    DevBuf<> dF, dA, dg;
    CFLX_TRY(stage(dF, a_n, F));
    CFLX_TRY(stage(dA, a_n, A));
    CFLX_TRY(stage(dg, 2 * (size_t)L.M));
    CFLX_TRY(equil_growth_cols(dF.as<double>(), dA.as<double>(), L, mode == 1, ncols, dg.as<double>(), 0));
    CFLX_TRY(fetch(amax_out, dg.p, L.M));
    CFLX_TRY(fetch(fmax_out, dg.as<double>() + L.M, L.M));
    CFLX_CUDA(cudaDeviceSynchronize());
    return CFLX_OK;
}

// the seed, scatter and zero-fill kernels of the inverse (inverse.cu) on one share
int cflx_dbg_inverse_share(int mode, const cflx_share_layout* share, int c0, int nc, int rows, const double* X, int ldx,
                           const int* perm, double* W_out, double* share_inout, int zero_fill) {
    CFLX_TRY(check_device());
    Layout L;
    CFLX_TRY(share_layout(__func__, share, TILED | COVERED, &L));
    REFUSE_IF(mode != 0 && mode != 1);
    REFUSE_IF(c0 < 0 || nc < 1 || c0 + nc > L.M);
    REFUSE_IF(rows < 0 || rows > L.Ml);
    REFUSE_IF(share_inout && (!X || (mode == 0 && !perm)));
    REFUSE_IF(share_inout && ldx < nc);
    const size_t w_n = (size_t)L.Ml * round_up(nc, 8);
    if (W_out) {
        DevBuf<> dW;
        CFLX_TRY(stage(dW, w_n));
        CFLX_CUDA(cudaMemset(dW.p, 0, sizeof(double) * w_n));
        CFLX_TRY(launch_inverse_seed(dW.as<double>(), (int)round_up(nc, 8), L, rows, c0, nc, 0));
        CFLX_TRY(fetch(W_out, dW.p, w_n));
    }
    if (share_inout) {
        const size_t a_n = (size_t)L.Ml * L.Nl;
        DevBuf<> dA, dX, dp;
        CFLX_TRY(stage(dA, a_n, share_inout));
        CFLX_TRY(stage(dX, (size_t)L.M * ldx, X));
        CFLX_TRY(stage(dp, L.M, mode == 0 ? perm : nullptr));
        CFLX_TRY(launch_inverse_scatter(mode == 0 ? InvKind::LU : InvKind::Chol, dX.as<double>(), ldx, c0, nc,
                                        mode == 0 ? dp.as<int>() : nullptr, L, dA.as<double>(), 0));
        if (mode == 1 && zero_fill) CFLX_TRY(launch_inverse_zero(L, dA.as<double>(), 0));
        CFLX_TRY(fetch(share_inout, dA.p, a_n));
    }
    CFLX_CUDA(cudaDeviceSynchronize());
    return CFLX_OK;
}

// the pack and scatter kernels of the distributed solves (solve_local.cu) on one right-hand side share
int cflx_dbg_solve_local_share(int mode, const cflx_share_layout* share, int nrhs, int c0, int w, const double* B, int ldb,
                               double* Bk_out, const double* Xk, double* X_inout, int ldx) {
    CFLX_TRY(check_device());
    Layout L;
    CFLX_TRY(share_layout(__func__, share, TILED, &L));
    const auto [M, v, Kappa, Ml, Nl, Px, Py, pi, pj] = *share;
    REFUSE_IF(mode != 0 && mode != 1);
    REFUSE_IF(M < (Ml / v) * Px * v);
    REFUSE_IF(nrhs < 1);
    REFUSE_IF(c0 < 0 || w < 1 || c0 + w > nrhs);
    REFUSE_IF(Nl != rhs_local_cols(nrhs, v, Py));
    REFUSE_IF(Bk_out && (!B || ldb < Nl));
    REFUSE_IF(X_inout && (!Xk || ldx < Nl));
    const int rows = solve_local_rows(L, mode == 1), ldn = (int)round_up(w, 8);
    const size_t k_n = (size_t)M * ldn;
    if (Bk_out) {
        DevBuf<> dB, dK;
        CFLX_TRY(stage(dB, (size_t)Ml * ldb, B));
        CFLX_TRY(stage(dK, k_n));
        CFLX_TRY(launch_solve_local_pack(dB.as<double>(), ldb, L, rows, c0, w, dK.as<double>(), ldn, 0));
        CFLX_TRY(fetch(Bk_out, dK.p, k_n));
    }
    if (X_inout) {
        DevBuf<> dX, dK;
        CFLX_TRY(stage(dX, (size_t)Ml * ldx, X_inout));
        CFLX_TRY(stage(dK, k_n, Xk));
        CFLX_TRY(launch_solve_local_scatter(dK.as<double>(), ldn, L, rows, c0, w, dX.as<double>(), ldx, 0));
        CFLX_TRY(fetch(X_inout, dX.p, (size_t)Ml * ldx));
    }
    CFLX_CUDA(cudaDeviceSynchronize());
    return CFLX_OK;
}

// the random butterfly transforms (rbt.cu) on one share, with the multipliers formed as cflx_lu_rbt forms them
int cflx_dbg_rbt_share(int op, const cflx_share_layout* share, int depth, const double* u, const double* v, int ncols,
                       double* share_inout, int ld) {
    CFLX_TRY(check_device());
    Layout L;
    CFLX_TRY(share_layout(__func__, share, op == 4 ? TILED | COVERED : TILED, &L));
    REFUSE_IF(op < 0 || op > 4);
    REFUSE_IF(depth < 1 || depth > 4);
    REFUSE_IF(L.Ml % (L.v << depth));
    REFUSE_IF(op == 4 && L.Nl % (L.v << depth));
    REFUSE_IF(op != 4 && L.M < (L.Ml / L.v) * L.Px * L.v);
    REFUSE_IF(op != 4 && ncols < 1);
    const int w = op == 4 ? L.Nl : ncols;
    REFUSE_IF(!share_inout || ld < w);
    REFUSE_IF(!u && op != 1 && op != 2);
    REFUSE_IF(!v && op != 0 && op != 3);
    const size_t n = (size_t)depth * L.M;
    std::vector<double> sc(2 * n, 0.0);
    if (u) rbt_scales(u, n, sc.data());
    if (v) rbt_scales(v, n, sc.data() + n);
    const size_t x_n = (size_t)L.Ml * ld;
    DevBuf<> dX, ds;
    CFLX_TRY(stage(dX, x_n, share_inout));
    CFLX_TRY(stage(ds, 2 * n, sc.data()));
    CFLX_TRY(launch_rbt((RbtOp)op, dX.as<double>(), ld, L, w, INT_MAX, depth, ds.as<double>(), ds.as<double>() + n, 0));
    CFLX_TRY(fetch(share_inout, dX.p, x_n));
    CFLX_CUDA(cudaDeviceSynchronize());
    return CFLX_OK;
}

// the sign pass between the sweeps of a signed Cholesky solve (solve.cu launch_solve_signs) on one share's Z
int cflx_dbg_solve_signs(const cflx_share_layout* share, int ldn, const double* sgn, double* Z_inout) {
    CFLX_TRY(check_device());
    Layout L;
    CFLX_TRY(share_layout(__func__, share, TILED, &L));
    REFUSE_IF(ldn < 1);
    REFUSE_IF(!sgn);
    REFUSE_IF(!Z_inout);
    const size_t n = (size_t)L.Nl * ldn;
    DevBuf<> dZ, ds;
    CFLX_TRY(stage(dZ, n, Z_inout));
    CFLX_TRY(stage(ds, (size_t)L.M, sgn));
    CFLX_TRY(launch_solve_signs(dZ.as<double>(), ldn, L, ds.as<double>(), 0));
    CFLX_TRY(fetch(Z_inout, dZ.p, n));
    CFLX_CUDA(cudaDeviceSynchronize());
    return CFLX_OK;
}

// the per-share passes of the 1-norm and the infinity-norm (norm.cu) on one layer-0 share: mode 0 the column sums, 1 the
// column sums of the symmetric matrix stored as its lower triangle, 2 the row sums
int cflx_dbg_norm_share(int mode, const cflx_share_layout* share, const double* A, double* out) {
    CFLX_TRY(check_device());
    Layout L;
    CFLX_TRY(share_layout(__func__, share, TILED | COVERED | NONEMPTY, &L));
    REFUSE_IF(mode < 0 || mode > 2);
    REFUSE_IF(!A || !out);
    int ncp = 0, nrp = 0;
    norm1_partials(L, &ncp, &nrp);
    DevBuf<> dA, dcol, drow, dout;
    CFLX_TRY(stage(dA, (size_t)L.Ml * L.Nl, A));
    CFLX_TRY(stage(dcol, (size_t)ncp * L.Nl));
    CFLX_TRY(stage(drow, (size_t)nrp * L.Ml));
    CFLX_TRY(stage(dout, L.M));
    double* o = dout.as<double>();
    if (mode == 2) {  // norminf_grid zeroes the vector; the column sums write every entry (NaN shows one they miss)
        CFLX_CUDA(cudaMemset(o, 0, sizeof(double) * L.M));
        CFLX_TRY(launch_norminf_share(dA.as<double>(), L, o, 0));
    } else {
        CFLX_TRY(launch_fill(o, L.M, std::numeric_limits<double>::quiet_NaN(), 0));
        CFLX_TRY(launch_norm1_share(dA.as<double>(), L, mode == 1, dcol.as<double>(), drow.as<double>(), o, 0));
    }
    CFLX_TRY(fetch(out, o, L.M));
    CFLX_CUDA(cudaDeviceSynchronize());
    return CFLX_OK;
}

// cflx_chol_validate's per-share kernels on one layer-0 share (each output may be null): the sum of squares of its lower
// triangle of the real tiles, and the masked transposed panel of step t
int cflx_dbg_chol_validate_share(const cflx_share_layout* share, const double* A, int t, double* PT_out, double* sumsq_out) {
    CFLX_TRY(check_device());
    Layout L;
    CFLX_TRY(share_layout(__func__, share, TILED | NONEMPTY, &L));
    const auto [M, v, Kappa, Ml, Nl, Px, Py, pi, pj] = *share;
    REFUSE_IF(M != std::max((Ml / v) * Px, (Nl / v) * Py) * v);
    REFUSE_IF(Kappa < 1);
    REFUSE_IF(!A);
    REFUSE_IF(t < 0 || t >= Kappa);
    REFUSE_IF((t / Py + 1) * v > Nl);
    const int64_t ldp = chol_panel_ld(Ml);
    DevBuf<> dA, dacc, dPT;
    CFLX_TRY(stage(dA, (size_t)Ml * Nl, A));
    CFLX_TRY(stage(dacc, 1 + SUMSQ_PARTIALS));
    CFLX_TRY(stage(dPT, v * ldp));
    if (sumsq_out) {
        double* acc = dacc.as<double>();
        CFLX_CUDA(cudaMemset(acc, 0, sizeof(double)));
        CFLX_TRY(launch_sumsq_lower(dA.as<double>(), L, acc + 1, acc, 0));
        CFLX_TRY(fetch(sumsq_out, acc, 1));
    }
    if (PT_out) {  // v x chol_panel_ld(Ml); NaN where the kernel writes nothing (and everywhere off grid column t % Py)
        CFLX_TRY(launch_fill(dPT.as<double>(), v * ldp, std::numeric_limits<double>::quiet_NaN(), 0));
        const int row0 = first_local_tile(t, pi, Px) * v;
        if (pj == t % Py)  // the guard and the arguments of cflx_chol_validate
            CFLX_TRY(launch_extract_l_panel_T(dA.as<double>(), Nl, row0, (t / Py) * v, Ml - row0, L, t, dPT.as<double>(),
                                              chol_piece_ld(L, t, pi), 0));
        CFLX_TRY(fetch(PT_out, dPT.p, v * ldp));
    }
    CFLX_CUDA(cudaDeviceSynchronize());
    return CFLX_OK;
}

// the two extract kernels of cflx_lu_validate's sweep, step t, on one layer-0 share C of the packed factors, under the
// owner guards of the sweep (each output may be null)
int cflx_dbg_lu_validate_share(const cflx_share_layout* share, const double* C, int t, double* LT_out, double* U_out) {
    CFLX_TRY(check_device());
    Layout L;
    CFLX_TRY(share_layout(__func__, share, TILED | NONEMPTY, &L));
    const auto [M, v, Kappa, Ml, Nl, Px, Py, pi, pj] = *share;
    REFUSE_IF((Ml / v) * Px != (Nl / v) * Py);  // the LU's shares of an M x M matrix
    REFUSE_IF(M != (Ml / v) * Px * v);
    REFUSE_IF(Kappa != M / v);
    REFUSE_IF(!C);
    REFUSE_IF(t < 0 || t >= Kappa);
    const int64_t ldp = round_up(Ml, 2);
    const double nan = std::numeric_limits<double>::quiet_NaN();
    DevBuf<> dC, dLT, dU;
    CFLX_TRY(stage(dC, (size_t)Ml * Nl, C));
    CFLX_TRY(stage(dLT, v * ldp));
    CFLX_TRY(stage(dU, (size_t)v * Nl));
    if (LT_out) {  // v x round_up(Ml, 2), NaN where the kernel writes nothing
        CFLX_TRY(launch_fill(dLT.as<double>(), v * ldp, nan, 0));
        CFLX_TRY(launch_lu_extract_l(dC.as<double>(), L, t, dLT.as<double>(), ldp, 0));
        CFLX_TRY(fetch(LT_out, dLT.p, v * ldp));
    }
    if (U_out) {  // v x Nl
        CFLX_TRY(launch_fill(dU.as<double>(), (int64_t)v * Nl, nan, 0));
        CFLX_TRY(launch_lu_extract_u(dC.as<double>(), L, t, dU.as<double>(), Nl, 0));
        CFLX_TRY(fetch(U_out, dU.p, (size_t)v * Nl));
    }
    CFLX_CUDA(cudaDeviceSynchronize());
    return CFLX_OK;
}

// the Cholesky update's column-operand gather (chol.cu) on one share at grid column pj, from the Px broadcast pieces of
// the panel of global tiles >= gfirst (host: piece p is v x chol_piece_ld(p), back to back), for the local column tiles
// with global index >= gfirst (Bc's tile t: local tile lj0 + t); Bc_out is v x Nl, NaN where nothing is written
int cflx_dbg_chol_gather_cols(const cflx_share_layout* share, int gfirst, const double* pieces, double* Bc_out) {
    CFLX_TRY(check_device());
    Layout L;
    CFLX_TRY(share_layout(__func__, share, TILED | NONEMPTY, &L));
    REFUSE_IF(gfirst < 0);
    REFUSE_IF(!pieces || !Bc_out);
    const int v = L.v, Ml = L.Ml, Nl = L.Nl, Px = L.Px, Py = L.Py, pj = L.pj;
    const int64_t ldp = chol_panel_ld(Ml), piece_stride = (int64_t)v * ldp, ldb = Nl;
    const double nan = std::numeric_limits<double>::quiet_NaN();
    DevBuf<> dG, dB;
    CFLX_TRY(stage(dG, Px * piece_stride));
    CFLX_TRY(stage(dB, v * ldb));
    CFLX_TRY(launch_fill(dG.as<double>(), Px * piece_stride, nan, 0));
    CFLX_TRY(launch_fill(dB.as<double>(), v * ldb, nan, 0));
    size_t off = 0;
    for (int p = 0; p < Px; ++p) {  // what broadcast_pieces sends: v chol_piece_ld doubles of the pieces with active rows
        const size_t n = (size_t)v * chol_piece_ld(L, gfirst, p);
        if (Ml - first_local_tile(gfirst, p, Px) * v > 0)
            CFLX_CUDA(cudaMemcpy(dG.as<double>() + p * piece_stride, pieces + off, sizeof(double) * n, cudaMemcpyHostToDevice));
        off += n;
    }
    const int lj0 = first_local_tile(gfirst, pj, Py), ntc = Nl / v - lj0;
    for (int t = 0; t < ntc; ++t) {  // every read of the kernel lies inside the Px piece slots
        const int j = (lj0 + t) * Py + pj, p = j % Px, first = first_local_tile(gfirst, p, Px);
        const int64_t ldg = std::max(2, (Ml - first * v + 1) & ~1);
        if (j / Px < first || p * piece_stride + (v - 1) * ldg + (int64_t)(j / Px - first + 1) * v > Px * piece_stride) {
            set_last_error("cflx_dbg_chol_gather_cols: refused, column tile %d reads outside the pieces", j);
            return CFLX_ERR_ARG;
        }
    }
    if (ntc > 0)
        CFLX_TRY(launch_gather_cols(dG.as<double>(), piece_stride, dB.as<double>(), ldb, v, Px, Py, pj, lj0, ntc, gfirst, Ml, 0));
    CFLX_TRY(fetch(Bc_out, dB.p, v * ldb));
    CFLX_CUDA(cudaDeviceSynchronize());
    return CFLX_OK;
}

// the refinement's assembly (refine.cu) from the host chunks of Px Py Pz ranks: mode 0 dgerfs' R, ratio and W; 1
// dla_lin_berr's R, ratio and Q; 2 the double-double R.  safe1, safe2 and nz eps are refine_safe's for M.
int cflx_dbg_refine_assemble(int mode, int Px, int Py, int Pz, int v, int M, int Ml, int Nl, int nn, int tn, int nrhs,
                             int ldn, const double* all, const double* B, double* R_out, double* ratio_out, double* W_out,
                             double* Q_out) {
    CFLX_TRY(check_device());
    REFUSE_IF(mode < 0 || mode > 2);
    REFUSE_IF(Px < 1 || Py < 1 || Pz < 1 || v < 1 || M < 1 || Ml < 0 || Nl < 0);
    REFUSE_IF(Ml % v || Nl % v);
    REFUSE_IF(!nn && !tn);
    REFUSE_IF(nrhs < 1 || ldn < nrhs);
    REFUSE_IF(!all || !B);
    REFUSE_IF((nn && M > (Ml / v) * Px * v) || (tn && M > (Nl / v) * Py * v));
    const int64_t chunk = (int64_t)((nn ? Ml : 0) + (tn ? Nl : 0)) * 2 * ldn, mat = (int64_t)M * ldn;
    const int64_t all_n = chunk * Px * Py * Pz;
    DevBuf<> dall, dB, dR, dratio, dW, dQ;
    CFLX_TRY(stage(dall, all_n, all));
    CFLX_TRY(stage(dB, mat, B));
    const double nan = std::numeric_limits<double>::quiet_NaN();
    for (DevBuf<>* b : {&dR, &dratio, &dW, &dQ}) {
        CFLX_TRY(stage(*b, mat));
        CFLX_TRY(launch_fill(b->as<double>(), mat, nan, 0));
    }
    double safe1, safe2, nzeps;
    refine_safe(M, &safe1, &safe2, &nzeps);
    AssembleArgs a{dall.as<double>(), chunk, Ml, Nl, ldn, nrhs, M, nn != 0, tn != 0, v, Px, Py, Pz, dB.as<double>(),
                   dR.as<double>(), dratio.as<double>(), mode == 1 ? nullptr : dW.as<double>(), safe1, safe2, nzeps};
    a.lin_berr = mode == 1;
    a.Q = mode == 1 ? dQ.as<double>() : nullptr;
    CFLX_TRY(launch_assemble(a, mode == 2, 0));
    CFLX_TRY(fetch(R_out, dR.p, mat));
    CFLX_TRY(fetch(ratio_out, dratio.p, mat));
    CFLX_TRY(fetch(W_out, dW.p, mat));
    CFLX_TRY(fetch(Q_out, dQ.p, mat));
    CFLX_CUDA(cudaDeviceSynchronize());
    return CFLX_OK;
}

// the refinement's per-column steps (refine.cu) on host M x ldn arrays A and D, nrhs columns, sel (ldn ints) the
// per-column selector; each output may be null: max_out (nrhs) column_max of A; stats_out (nrhs x 5) column_stats of
// y = A, dy = D (d: M scales or null); select_out select_cols of A; add_out add_cols of D into A; Y_out / T_inout
// update_x of (A, T_inout) by D with how = sel
int cflx_dbg_refine_columns(int M, int ldn, int nrhs, const double* A, const double* D, const double* d, const int* sel,
                            double* max_out, double* stats_out, double* select_out, double* add_out, double* Y_out,
                            double* T_inout) {
    CFLX_TRY(check_device());
    REFUSE_IF(M < 1 || nrhs < 1 || ldn < nrhs);
    REFUSE_IF(!A);
    REFUSE_IF((stats_out || add_out || Y_out) && !D);
    REFUSE_IF((select_out || add_out || Y_out) && !sel);
    REFUSE_IF(!Y_out != !T_inout);
    const int64_t mat = (int64_t)M * ldn;
    DevBuf<> dA, dD, dd, dsel, dW, dT, dv;
    CFLX_TRY(stage(dA, mat, A));
    CFLX_TRY(stage(dD, mat, D));
    CFLX_TRY(stage(dd, M, d));
    CFLX_TRY(stage(dsel, ldn, sel));
    CFLX_TRY(stage(dW, mat));
    CFLX_TRY(stage(dT, mat, T_inout));
    CFLX_TRY(stage(dv, (size_t)nrhs * REFINE_NSTAT));
    const double* a = dA.as<double>();
    double* w = dW.as<double>();
    if (max_out) CFLX_TRY(launch_column_max(a, M, ldn, nrhs, dv.as<double>(), 0));
    CFLX_TRY(fetch(max_out, dv.p, nrhs));
    if (stats_out)
        CFLX_TRY(launch_column_stats(a, dD.as<double>(), d ? dd.as<double>() : nullptr, M, ldn, nrhs, dv.as<double>(), 0));
    CFLX_TRY(fetch(stats_out, dv.p, (size_t)nrhs * REFINE_NSTAT));
    if (select_out) {
        CFLX_TRY(launch_fill(w, mat, std::numeric_limits<double>::quiet_NaN(), 0));
        CFLX_TRY(launch_select_cols(a, dsel.as<int>(), M, ldn, w, 0));
        CFLX_TRY(fetch(select_out, w, mat));
    }
    if (add_out) {
        CFLX_CUDA(cudaMemcpy(w, a, sizeof(double) * mat, cudaMemcpyDeviceToDevice));
        CFLX_TRY(launch_add_cols(w, dD.as<double>(), dsel.as<int>(), M, ldn, 0));
        CFLX_TRY(fetch(add_out, w, mat));
    }
    if (Y_out) {
        CFLX_CUDA(cudaMemcpy(w, a, sizeof(double) * mat, cudaMemcpyDeviceToDevice));
        CFLX_TRY(launch_update_x(w, dT.as<double>(), dD.as<double>(), dsel.as<int>(), M, ldn, 0));
        CFLX_TRY(fetch(Y_out, w, mat));
        CFLX_TRY(fetch(T_inout, dT.p, mat));
    }
    CFLX_CUDA(cudaDeviceSynchronize());
    return CFLX_OK;
}

// the determinant's product kernel (det.cu) on host vectors
int cflx_dbg_det(int n, const double* d, const double* s1, const double* s2, int square, double* mant_out,
                 int64_t* exp_out, int* neg_out, int* first_zero_out, int* nonfinite_out) {
    CFLX_TRY(check_device());
    REFUSE_IF(n < 1);
    REFUSE_IF(!d);
    REFUSE_IF(square != 0 && square != 1);
    DevBuf<> dd, ds1, ds2, dr;
    CFLX_TRY(stage(dd, n, d));
    CFLX_TRY(stage(ds1, n, s1));
    CFLX_TRY(stage(ds2, n, s2));
    CFLX_TRY(stage<DetResult>(dr, 1));
    CFLX_TRY(launch_det(dd.as<double>(), s1 ? ds1.as<double>() : nullptr, s2 ? ds2.as<double>() : nullptr, n, square != 0,
                        dr.as<DetResult>(), 0));
    DetResult r{};
    CFLX_TRY(fetch(&r, dr.p, 1));
    if (mant_out) *mant_out = r.mant;
    if (exp_out) *exp_out = r.exp;
    if (neg_out) *neg_out = r.neg;
    if (first_zero_out) *first_zero_out = r.first_zero;
    if (nonfinite_out) *nonfinite_out = r.nonfinite;
    return CFLX_OK;
}

// the residual kernels of the refinement (refine.cu) on one layer-0 share
int cflx_dbg_residual(int mode, const cflx_share_layout* share, const double* A, int nrhs, const double* Xc,
                      const double* Xr, double* P_out, double* Q_out, int reps, double* ms_out) {
    CFLX_TRY(check_device());
    Layout L;  // M unused: the kernels index by local row and column only
    CFLX_TRY(share_layout(__func__, share, 0, &L));
    REFUSE_IF(mode < 0 || mode > 2);
    REFUSE_IF(L.v & 3);
    REFUSE_IF(L.Nl & 1);
    REFUSE_IF(nrhs < 1);
    REFUSE_IF(!A || (mode != 1 && !Xc) || (mode != 0 && !Xr));
    return residual_run(mode, L, A, nrhs, Xc, Xr, P_out, Q_out, reps, ms_out,
                        [&](ResidMode m, const double* a, const double* xc, const double* xr, double* p, double* q) {
                            return launch_residual(m, a, L, xc, xr, nrhs, nrhs, p, q, nrhs, 0);
                        });
}

int cflx_dbg_residual_x(int mode, const cflx_share_layout* share, const double* A, int nrhs, const double* Xc,
                        const double* Xct, const double* Xr, const double* Xrt, double* hi_out, double* lo_out, int reps,
                        double* ms_out) {
    CFLX_TRY(check_device());
    Layout L;  // M unused, as in cflx_dbg_residual
    CFLX_TRY(share_layout(__func__, share, 0, &L));
    REFUSE_IF(mode < 0 || mode > 2);
    REFUSE_IF(nrhs < 1);
    REFUSE_IF(!A || (mode != 1 && !Xc) || (mode != 0 && !Xr));
    DevBuf<> dXct, dXrt;
    CFLX_TRY(stage(dXct, (size_t)L.Nl * nrhs, Xct));
    CFLX_TRY(stage(dXrt, (size_t)L.Ml * nrhs, Xrt));
    return residual_run(mode, L, A, nrhs, Xc, Xr, hi_out, lo_out, reps, ms_out,
                        [&](ResidMode m, const double* a, const double* xc, const double* xr, double* hi, double* lo) {
                            return launch_residual_x(m, a, L, xc, Xct ? dXct.as<double>() : nullptr, xr,
                                                     Xrt ? dXrt.as<double>() : nullptr, nrhs, nrhs, hi, lo, nrhs, 0);
                        });
}

int cflx_dbg_panel(int n, int v, const double* panel, int* perm_out, double* A00_out, double* LU_out, int reps,
                   double* ms_out) {
    CFLX_TRY(check_device());
    REFUSE_IF(n < 0 || v <= 0);
    const int64_t ld = std::max<int64_t>(2, round_up(n, 2));
    // host transpose into the kernel's K-major layout
    std::vector<double> WT((size_t)v * ld, 0.0);
    for (int r = 0; r < n; ++r)
        for (int c = 0; c < v; ++c) WT[(size_t)c * ld + r] = panel[(size_t)r * v + c];
    DevBuf<> dW, dW0, dA00, dA00T, dperm;
    CFLX_TRY(stage(dW, WT.size()));
    CFLX_TRY(stage(dW0, WT.size(), WT.data()));
    CFLX_TRY(stage(dA00, (size_t)v * v));
    CFLX_TRY(stage(dA00T, (size_t)v * v));
    CFLX_TRY(stage<int>(dperm, 2 * (size_t)v));
    CFLX_CUDA(cudaMemset(dA00.p, 0, sizeof(double) * v * v));
    Events<2> ev;
    CFLX_TRY(ev.create());
    PanelWorkspace ws{};
    CFLX_TRY(panel_workspace_create(&ws));
    if (const char* e = getenv("CFLX_PANEL_CTAS")) ws.cta_cap = atoi(e);  // time the search on the look-ahead's SM budget
    if (reps < 1) reps = 1;
    float total = 0;
    int nb = 0, rc = CFLX_OK;
    for (int r = 0; r < reps + 1 && rc == CFLX_OK; ++r) {
        cudaMemcpyAsync(dW.p, dW0.p, sizeof(double) * v * ld, cudaMemcpyDeviceToDevice, 0);
        cudaEventRecord(ev[0]);
        rc = launch_panel_getrf_a00(dW.as<double>(), ld, n, v, dperm.as<int>(), dA00.as<double>(), &nb, &ws, 0);
        cudaEventRecord(ev[1]);
        if (cudaEventSynchronize(ev[1]) != cudaSuccess) rc = CFLX_ERR_CUDA;
        float ms = 0;
        cudaEventElapsedTime(&ms, ev[0], ev[1]);
        if (r > 0) total += ms;
    }
    if (rc == CFLX_OK && n >= v)
        rc = launch_gather_a00(dW.as<double>(), ld, dperm.as<int>(), v, nb, dA00.as<double>(), dA00T.as<double>(), 0);
    if (rc != CFLX_OK) {
        if (rc == CFLX_ERR_CUDA) set_last_error("panel kernel failed: %s", cudaGetErrorString(cudaGetLastError()));
        return rc;
    }
    if (ms_out) *ms_out = total / reps;
    CFLX_TRY(fetch(perm_out, dperm.p, v));
    CFLX_TRY(fetch(A00_out, dA00.p, (size_t)v * v));
    if (LU_out) {
        CFLX_TRY(fetch(WT.data(), dW.p, WT.size()));
        for (int r = 0; r < n; ++r)
            for (int c = 0; c < v; ++c) LU_out[(size_t)r * v + c] = WT[(size_t)c * ld + r];
    }
    CFLX_CUDA(cudaDeviceSynchronize());
    return CFLX_OK;
}

int cflx_dbg_trsm(int n, int v, int nb, int64_t ld, const double* A00, const double* B, double* X_out, const double* R,
                  double* Y_out) {
    CFLX_TRY(check_device());
    REFUSE_IF(n <= 0 || v <= 0 || v % 4 != 0);
    if (nb == 0)
        for (int c : {128, 64, 32, 16, 8, 4})
            if (!nb && v % c == 0) nb = c;
    if (nb != 4 && nb != 8 && nb != 16 && nb != 32 && nb != 64 && nb != 128)
        return refuse(__func__, "nb not 4, 8, 16, 32, 64 or 128", CFLX_ERR_UNSUPPORTED);
    REFUSE_IF(v % nb != 0);
    if (ld == 0) ld = round_up(n, 2);
    REFUSE_IF((ld & 1) || ld < round_up(n, 2));
    // the padding columns [n, ld) of the operand panels hold NaN: they must not reach the n solved columns
    const double nan = std::numeric_limits<double>::quiet_NaN();
    std::vector<double> A00T((size_t)v * v), BT((size_t)v * ld, nan), RT((size_t)v * ld, nan);
    for (int i = 0; i < v; ++i)
        for (int j = 0; j < v; ++j) A00T[(size_t)j * v + i] = A00[(size_t)i * v + j];
    const size_t vv = (size_t)v * v, panel = (size_t)v * ld;
    DevBuf<> dA, dAT, dUinv, dLinvT;
    CFLX_TRY(stage(dA, vv, A00));
    CFLX_TRY(stage(dAT, vv, A00T.data()));
    CFLX_TRY(stage(dUinv, vv));
    CFLX_TRY(stage(dLinvT, vv));
    CFLX_TRY(launch_diag_inverses(dA.as<double>(), v, nb, dUinv.as<double>(), dLinvT.as<double>(), 0));
    if (B && X_out) {  // X = B * U^-1, B is n x v row-major
        for (int r = 0; r < n; ++r)
            for (int c = 0; c < v; ++c) BT[(size_t)c * ld + r] = B[(size_t)r * v + c];
        DevBuf<> dP, dL;
        CFLX_TRY(stage(dP, panel, BT.data()));
        CFLX_TRY(stage(dL, panel));
        CFLX_CUDA(cudaMemset(dL.p, 0, 8 * panel));
        CFLX_TRY(trsm_right_upper_T(dA.as<double>(), dUinv.as<double>(), v, nb, dP.as<double>(), dL.as<double>(), ld, n, 0));
        CFLX_TRY(fetch(BT.data(), dL.p, panel));
        for (int r = 0; r < n; ++r)
            for (int c = 0; c < v; ++c) X_out[(size_t)r * v + c] = BT[(size_t)c * ld + r];
    }
    if (R && Y_out) {  // Y = L^-1 * R, R is v x n row-major
        for (int i = 0; i < v; ++i)
            for (int c = 0; c < n; ++c) RT[(size_t)i * ld + c] = R[(size_t)i * n + c];
        DevBuf<> dR, dU;
        CFLX_TRY(stage(dR, panel, RT.data()));
        CFLX_TRY(stage(dU, panel));
        CFLX_CUDA(cudaMemset(dU.p, 0, 8 * panel));
        CFLX_TRY(trsm_left_lower_unit(dAT.as<double>(), dLinvT.as<double>(), v, nb, dR.as<double>(), dU.as<double>(), ld,
                                      (int)round_up(n, 2), 0));
        CFLX_TRY(fetch(RT.data(), dU.p, panel));
        for (int i = 0; i < v; ++i)
            for (int c = 0; c < n; ++c) Y_out[(size_t)i * n + c] = RT[(size_t)i * ld + c];
    }
    CFLX_CUDA(cudaDeviceSynchronize());
    return CFLX_OK;
}

// inverses of the nb x nb diagonal blocks of the v x v row-major A00 = L\U: Uinv_out / LinvT_out are [v / nb][nb][nb]
int cflx_dbg_diag_inverse(int v, int nb, const double* A00, double* Uinv_out, double* LinvT_out) {
    CFLX_TRY(check_device());
    REFUSE_IF(v <= 0 || nb <= 0 || v % nb != 0);
    REFUSE_IF(!A00);
    const size_t vv = (size_t)v * v, blocks = (size_t)v * nb;
    DevBuf<> dA, dU, dL;
    CFLX_TRY(stage(dA, vv, A00));
    CFLX_TRY(stage(dU, blocks));
    CFLX_TRY(stage(dL, blocks));
    CFLX_TRY(launch_diag_inverses(dA.as<double>(), v, nb, dU.as<double>(), dL.as<double>(), 0));
    CFLX_TRY(fetch(Uinv_out, dU.p, blocks));
    CFLX_TRY(fetch(LinvT_out, dL.p, blocks));
    CFLX_CUDA(cudaDeviceSynchronize());
    return CFLX_OK;
}

// Cholesky of one v x v row-major tile A (lower triangle read) on the kernels of the factorisation.  variant 0: the
// one-CTA potrf_tile_kernel (4 <= v <= 512); 1: potrf128_kernel (v == 128); 2: the 128-block driver potrf_tile()
// (v % 128 == 0, v >= 256).  L_out = L (zeros above the diagonal), LT_out = L^T, info_out = 1 + first failing column or 0.
int cflx_dbg_potrf_tile(int v, const double* A, double* L_out, double* LT_out, int* info_out, int variant) {
    CFLX_TRY(check_device());
    REFUSE_IF(!A);
    REFUSE_IF(variant < 0 || variant > 2);
    REFUSE_IF(v < 4 || v > 512 || (variant == 1 && v != 128) || (variant == 2 && potrf_tile_scratch(v) == 0));
    const size_t vv = (size_t)v * v;
    DevBuf<> dD, dUT, dUc, dQ, dinfo;
    CFLX_TRY(stage(dD, vv, A));
    CFLX_TRY(stage(dUT, vv));
    CFLX_TRY(stage(dUc, vv));
    CFLX_TRY(stage<int>(dinfo, 1));
    if (variant == 2) CFLX_TRY(stage(dQ, potrf_tile_scratch(v)));
    CFLX_CUDA(cudaMemset(dUT.p, 0, 8 * vv));
    CFLX_CUDA(cudaMemset(dinfo.p, 0, sizeof(int)));
    CFLX_TRY(potrf_setup(v));
    int64_t launches = 0;
    if (variant == 1)
        CFLX_TRY(potrf_block128(dD.as<double>(), v, dUT.as<double>(), v, dUc.as<double>(), dinfo.as<int>(), 0, 0));
    else
        CFLX_TRY(potrf_tile(dD.as<double>(), dUT.as<double>(), dQ.as<double>(), dinfo.as<int>(), 0, v, 0, &launches));
    CFLX_TRY(fetch(L_out, dD.p, vv));
    CFLX_TRY(fetch(LT_out, dUT.p, vv));
    CFLX_TRY(fetch(info_out, dinfo.p, 1));
    CFLX_CUDA(cudaDeviceSynchronize());
    return CFLX_OK;
}

// The signed Cholesky of one tile on the kernels of cflx_chol_factor_ldlt, variants as cflx_dbg_potrf_tile
int cflx_dbg_ldlt_tile(int v, const double* A, double tiny, double* R_out, double* SRT_out, double* s_out, int* nrepl_out,
                       int* inertia_out, int* info_out, int variant) {
    CFLX_TRY(check_device());
    REFUSE_IF(!A);
    REFUSE_IF(!(tiny >= 0.0));
    REFUSE_IF(variant < 0 || variant > 2);
    REFUSE_IF(v < 4 || v > 512 || (variant == 1 && v != 128) || (variant == 2 && potrf_tile_scratch(v) == 0));
    const size_t vv = (size_t)v * v;
    DevBuf<> dD, dUT, dUc, dQ, dinfo, dcnt, dsg;
    CFLX_TRY(stage(dD, vv, A));
    CFLX_TRY(stage(dUT, vv));
    CFLX_TRY(stage(dUc, vv));
    CFLX_TRY(stage(dsg, (size_t)v));
    CFLX_TRY(stage<int>(dinfo, 1));
    CFLX_TRY(stage<int>(dcnt, 4));
    if (variant == 2) CFLX_TRY(stage(dQ, potrf_tile_scratch(v)));
    CFLX_CUDA(cudaMemset(dUT.p, 0, 8 * vv));
    CFLX_CUDA(cudaMemset(dinfo.p, 0, sizeof(int)));
    CFLX_CUDA(cudaMemset(dcnt.p, 0, 4 * sizeof(int)));
    CFLX_TRY(potrf_setup(v));
    const LdltArgs sa{tiny, dsg.as<double>(), dcnt.as<int>()};
    int64_t launches = 0;
    if (variant == 1)
        CFLX_TRY(potrf_block128(dD.as<double>(), v, dUT.as<double>(), v, dUc.as<double>(), dinfo.as<int>(), 0, 0, &sa));
    else
        CFLX_TRY(potrf_tile(dD.as<double>(), dUT.as<double>(), dQ.as<double>(), dinfo.as<int>(), 0, v, 0, &launches, &sa));
    int cnt[4];
    CFLX_TRY(fetch(R_out, dD.p, vv));
    CFLX_TRY(fetch(SRT_out, dUT.p, vv));
    CFLX_TRY(fetch(s_out, dsg.p, (size_t)v));
    CFLX_TRY(fetch(cnt, dcnt.p, 4));
    CFLX_TRY(fetch(info_out, dinfo.p, 1));
    CFLX_CUDA(cudaDeviceSynchronize());
    if (nrepl_out) *nrepl_out = cnt[0];
    if (inertia_out)
        for (int i = 0; i < 3; ++i) inertia_out[i] = cnt[1 + i];
    return CFLX_OK;
}

// unpivoted LU of one v x v row-major block as cflx_lu_factor_fixed runs it: variant 0 the one-CTA kernel on the whole
// block, 1 the 128-block driver (v % 128 == 0, v >= 256; what the factorisation runs there)
int cflx_dbg_getrf_nopiv_tile(int v, const double* A, double tiny, double* LU_out, int* nrepl_out, int* info_out,
                              int variant) {
    CFLX_TRY(check_device());
    REFUSE_IF(!A || !LU_out || !info_out);
    REFUSE_IF(variant != 0 && variant != 1);
    REFUSE_IF(v < 4 || v > 1024 || v % 4 != 0);
    REFUSE_IF(variant == 1 && !getrf_nopiv_blocked(v));
    REFUSE_IF(!(tiny >= 0.0));
    const size_t vv = (size_t)v * v;
    std::vector<double> At(vv);  // the tile takes the block transposed, as the gather leaves it
    for (int i = 0; i < v; ++i)
        for (int c = 0; c < v; ++c) At[(size_t)c * v + i] = A[(size_t)i * v + c];
    DevBuf<> dB, dA, drec, dws;
    CFLX_TRY(stage(dB, vv, At.data()));
    CFLX_TRY(stage(dA, vv));
    CFLX_TRY(stage<int>(drec, 4));
    const size_t ws = getrf_nopiv_scratch(v, variant == 1);
    if (ws) CFLX_TRY(stage(dws, ws));
    CFLX_CUDA(cudaMemset(drec.p, 0, 4 * sizeof(int)));
    if (variant == 1) CFLX_TRY(gemm_tn_setup());
    int64_t launches = 0;
    CFLX_TRY(launch_getrf_nopiv_tile(dB.as<double>(), v, tiny, dA.as<double>(), nullptr, nullptr, nullptr, drec.as<int>(),
                                     0, variant == 1, ws ? dws.as<double>() : nullptr, 0, &launches));
    int rec[4];
    CFLX_TRY(fetch(LU_out, dA.p, vv));
    CFLX_TRY(fetch(rec, drec.p, 4));
    CFLX_CUDA(cudaDeviceSynchronize());
    if (nrepl_out) *nrepl_out = rec[0];
    *info_out = rec[1];
    return CFLX_OK;
}

// step 2 of the LU loop in isolation on ONE rank (Px = 1): plan_moves (analyze_pivots) + push_phase1..3 (push_pivots_up,
// conflux_opt.hpp:176-218) + the gri/igri bookkeeping, on an n_rows x n_cols row-major matrix (n_cols even).  The npiv
// pivot rows (local indices >= fnpr, tournament order) end up in rows [fnpr, fnpr+npiv) in that order.
// gri_out[n_rows] (optional) = new row -> old row.  a01_out (optional, npiv x n_cols) = the pivot rows phase 1 extracts.
int cflx_dbg_push_pivots(int n_rows, int n_cols, double* A_inout, int npiv, const int* pivot_rows, int fnpr, int* gri_out,
                         double* a01_out) {
    CFLX_TRY(check_device());
    REFUSE_IF(n_rows <= 0 || n_cols <= 0 || (n_cols & 1));
    REFUSE_IF(npiv < 0 || fnpr < 0 || npiv > n_rows - fnpr);
    if (npiv == 0) {
        if (gri_out) for (int i = 0; i < n_rows; ++i) gri_out[i] = i;
        return CFLX_OK;
    }
    REFUSE_IF(!A_inout || !pivot_rows);
    const int v = npiv;  // every pivot of the "tile" lives on this rank
    const size_t a_n = (size_t)n_rows * n_cols;
    DevBuf<> dA, dtmp, da01, dplan, dgp, dgri, dgrit, digri;
    CFLX_TRY(stage(dA, a_n, A_inout));
    CFLX_TRY(stage(dtmp, (size_t)v * n_cols));
    CFLX_TRY(stage(da01, (size_t)v * n_cols));
    CFLX_TRY(stage<int>(dplan, 6 * (size_t)v + 8 + n_rows));
    CFLX_TRY(stage(dgp, v, pivot_rows));
    CFLX_TRY(stage<int>(dgri, n_rows));
    CFLX_TRY(stage<int>(dgrit, n_rows));
    CFLX_TRY(stage<int>(digri, n_rows));
    MovePlan plan{};
    int* pm = dplan.as<int>();
    plan.npiv = pm; plan.nel = pm + 4; pm += 8;
    plan.cur_piv = pm; pm += v;
    plan.order = pm; pm += v;
    plan.slot2piv = pm; pm += v;
    plan.early = pm; pm += v;
    plan.late = pm; pm += 2 * v;
    plan.rowsrc = pm;
    // gri = identity with "tile size" n_rows so that global id == local row (Px = 1)
    CFLX_TRY(launch_iota_gri(dgri.as<int>(), digri.as<int>(), n_rows, n_rows, 1, 0, 0));
    // plan_moves maps a global id g to the local slot (g / (v*Px))*v + g % v: with v := n_rows that is g itself
    CFLX_TRY(launch_plan_moves(dgp.as<int>(), v, 1, 0, fnpr, n_rows, digri.as<int>(), plan, 0));
    CFLX_TRY(launch_push_phase1(dA.as<double>(), n_cols, n_cols, 0, plan, v, dtmp.as<double>(), da01.as<double>(), n_cols, 0, 0));
    CFLX_TRY(launch_push_phase2(dA.as<double>(), n_cols, n_cols, 0, plan, v, 0));
    CFLX_TRY(launch_push_phase3(dA.as<double>(), n_cols, n_cols, 0, fnpr, plan, v, dtmp.as<double>(), 0));
    CFLX_TRY(launch_update_gri(dgri.as<int>(), dgrit.as<int>(), digri.as<int>(), plan.rowsrc, fnpr, n_rows, n_rows, 1, 0));
    CFLX_TRY(fetch(A_inout, dA.p, a_n));
    CFLX_TRY(fetch(gri_out, dgri.p, n_rows));
    CFLX_TRY(fetch(a01_out, da01.p, (size_t)v * n_cols));
    CFLX_CUDA(cudaDeviceSynchronize());
    return CFLX_OK;
}

// D = C - AT^T * B on the int8 wgmma path (ozaki.cu): AT [K x M], B [K x N], C/D [M x N] row-major dense host arrays,
// K a multiple of 128, N even.  Optional outputs for tests: the digit planes [8][M][K] / [8][N][K] (int8) and the
// exponents [M] / [N], exactly as the kernels produced them.  ms_out = mean device time of the GEMM kernel alone.
int cflx_dbg_ozaki_gemm(int M, int N, int K, int row0, int col0, int max_ctas, const double* AT, const double* B,
                        const double* C, double* D, signed char* planesA_out, signed char* planesB_out, int* ea_out,
                        int* eb_out, int reps, double* ms_out, double* split_ms_out) {
    CFLX_TRY(check_device());
    REFUSE_IF(M <= 0 || N <= 0 || K <= 0 || (N & 1));
    REFUSE_IF(row0 < 0 || col0 < 0 || max_ctas < 0);
    REFUSE_IF(!AT || !B);
    // AT holds row0 + M operand rows, B col0 + N columns; the planes of all of them are made (B's in the two windows
    // [0, col0) and [col0, col0 + N), as the factorisation's look-ahead splits them), the product reads the window
    const int Ma = row0 + M, Nb = col0 + N;
    const int64_t ldat = round_up(Ma, 2), ldb = Nb, ldc = N;
    const size_t c_n = (size_t)M * ldc;
    DevBuf<> dA, dB, dC, dC0;
    CFLX_TRY(stage(dA, K * ldat));
    CFLX_TRY(stage(dB, K * ldb, B));
    CFLX_TRY(stage(dC, c_n));
    CFLX_TRY(stage(dC0, c_n, C));
    CFLX_CUDA(cudaMemset(dA.p, 0, sizeof(double) * K * ldat));
    CFLX_CUDA(cudaMemcpy2D(dA.p, ldat * 8, AT, (size_t)Ma * 8, (size_t)Ma * 8, K, cudaMemcpyHostToDevice));
    if (!C) CFLX_CUDA(cudaMemset(dC0.p, 0, sizeof(double) * c_n));
    Events<3> ev;
    CFLX_TRY(ev.create());
    OzakiWorkspace ws;
    int rc = ozaki_workspace_create(&ws, Ma, Nb, K);
    if (reps < 1) reps = 1;
    float ms = 0, ms_split = 0;
    for (int r = 0; r < reps + 1 && rc == CFLX_OK; ++r) {
        cudaMemcpyAsync(dC.p, dC0.p, sizeof(double) * c_n, cudaMemcpyDeviceToDevice, 0);
        cudaEventRecord(ev[0]);
        rc = ozaki_split_a(&ws, dA.as<double>(), ldat, Ma, 0);
        if (!rc && col0 > 0) rc = ozaki_split_b(&ws, dB.as<double>(), ldb, 0, col0, 0);
        if (!rc) rc = ozaki_split_b(&ws, dB.as<double>(), ldb, col0, N, 0);
        cudaEventRecord(ev[1]);
        if (!rc) rc = launch_ozaki_gemm(&ws, M, N, row0, col0, dC.as<double>(), ldc, max_ctas, 0);
        cudaEventRecord(ev[2]);
        if (cudaEventSynchronize(ev[2]) != cudaSuccess) {
            set_last_error("ozaki kernel failed: %s", cudaGetErrorString(cudaGetLastError()));
            rc = CFLX_ERR_CUDA;
        }
        float a = 0, b = 0;
        cudaEventElapsedTime(&a, ev[0], ev[1]);
        cudaEventElapsedTime(&b, ev[1], ev[2]);
        if (r > 0) {
            ms_split += a;
            ms += b;
        }
    }
    if (rc == CFLX_OK) rc = fetch(D, dC.p, c_n);
    for (int s = 0; s < 8 && rc == CFLX_OK; ++s) {
        if (planesA_out) rc = fetch(planesA_out + (size_t)s * Ma * K, ws.planesA + (size_t)s * ws.cap_a * K, (size_t)Ma * K);
        if (planesB_out && rc == CFLX_OK)
            rc = fetch(planesB_out + (size_t)s * Nb * K, ws.planesB + (size_t)s * ws.cap_b * K, (size_t)Nb * K);
    }
    if (rc == CFLX_OK) rc = fetch(ea_out, ws.ea, Ma);
    if (rc == CFLX_OK) rc = fetch(eb_out, ws.eb, Nb);
    if (rc == CFLX_OK && cudaDeviceSynchronize() != cudaSuccess) rc = CFLX_ERR_CUDA;
    if (ms_out) *ms_out = ms / reps;
    if (split_ms_out) *split_ms_out = ms_split / reps;
    return rc;
}

// D = C - AT^T * B on the TF32 wgmma path (tf32.cu): the split of every operand row, then one launch of the product
int cflx_dbg_gemm_tf32(int terms, int M, int N, int K, int row0, int col0, int max_ctas, const double* AT, const double* B,
                       const double* C, double* D, float* hiA_out, float* loA_out, float* hiB_out, float* loB_out,
                       int* ea_out, int* eb_out, int reps, double* ms_out, double* split_ms_out) {
    CFLX_TRY(check_device());
    REFUSE_IF(terms != 1 && terms != 3);
    REFUSE_IF(M <= 0 || N <= 0 || K <= 0);
    REFUSE_IF(row0 < 0 || col0 < 0 || max_ctas < 0);
    REFUSE_IF(!AT || !B || !D);
    const int Ma = row0 + M, Nb = col0 + N;
    const int64_t ldat = Ma, ldb = Nb, ldc = round_up(N, 2);
    DevBuf<> dA, dB, dC, dC0;
    CFLX_TRY(stage(dA, K * ldat, AT));
    CFLX_TRY(stage(dB, K * ldb, B));
    CFLX_TRY(stage(dC, (size_t)M * ldc));
    CFLX_TRY(stage(dC0, (size_t)M * ldc));
    CFLX_CUDA(cudaMemset(dC0.p, 0, sizeof(double) * M * ldc));
    if (C) CFLX_CUDA(cudaMemcpy2D(dC0.p, ldc * 8, C, (size_t)N * 8, (size_t)N * 8, M, cudaMemcpyHostToDevice));
    Events<3> ev;
    CFLX_TRY(ev.create());
    Tf32Workspace ws;
    int rc = tf32_workspace_create(&ws, Ma, Nb, K);
    if (reps < 1) reps = 1;
    float ms = 0, ms_split = 0;
    for (int r = 0; r < reps + 1 && rc == CFLX_OK; ++r) {
        cudaMemcpyAsync(dC.p, dC0.p, sizeof(double) * M * ldc, cudaMemcpyDeviceToDevice, 0);
        cudaEventRecord(ev[0]);
        rc = tf32_split_a(&ws, terms, dA.as<double>(), ldat, Ma, 0);
        if (!rc && col0 > 0) rc = tf32_split_b(&ws, terms, dB.as<double>(), ldb, 0, col0, 0);
        if (!rc) rc = tf32_split_b(&ws, terms, dB.as<double>(), ldb, col0, N, 0);
        cudaEventRecord(ev[1]);
        if (!rc) rc = launch_tf32_gemm(&ws, terms, M, N, row0, col0, dC.as<double>(), ldc, max_ctas, 0);
        cudaEventRecord(ev[2]);
        if (cudaEventSynchronize(ev[2]) != cudaSuccess) {
            set_last_error("tf32 kernel failed: %s", cudaGetErrorString(cudaGetLastError()));
            rc = CFLX_ERR_CUDA;
        }
        float a = 0, b = 0;
        cudaEventElapsedTime(&a, ev[0], ev[1]);
        cudaEventElapsedTime(&b, ev[1], ev[2]);
        if (r > 0) {
            ms_split += a;
            ms += b;
        }
    }
    if (rc == CFLX_OK && cudaMemcpy2D(D, (size_t)N * 8, dC.p, ldc * 8, (size_t)N * 8, M, cudaMemcpyDeviceToHost) != cudaSuccess)
        rc = CFLX_ERR_CUDA;
    const size_t na = (size_t)Ma * ws.KP, nb = (size_t)Nb * ws.KP;
    if (rc == CFLX_OK) rc = fetch(hiA_out, ws.hiA.p, na);
    if (rc == CFLX_OK && terms == 3) rc = fetch(loA_out, ws.loA.p, na);
    if (rc == CFLX_OK) rc = fetch(hiB_out, ws.hiB.p, nb);
    if (rc == CFLX_OK && terms == 3) rc = fetch(loB_out, ws.loB.p, nb);
    if (rc == CFLX_OK) rc = fetch(ea_out, ws.ea, Ma);
    if (rc == CFLX_OK) rc = fetch(eb_out, ws.eb, Nb);
    if (rc == CFLX_OK && cudaDeviceSynchronize() != cudaSuccess) rc = CFLX_ERR_CUDA;
    if (ms_out) *ms_out = ms / reps;
    if (split_ms_out) *split_ms_out = ms_split / reps;
    return rc;
}

// raw int8 tensor-core rate of back-to-back wgmma 64 x n x 32 instructions (two warpgroups per CTA, one CTA per SM,
// operands resident in shared memory).  Returns tera-MACs per second (x2 = TOP/s).
int cflx_dbg_wgmma_peak(int n, double* tmacs_out) {
    CFLX_TRY(check_device());
    REFUSE_IF(!tmacs_out);
    return wgmma_peak_probe(n, tmacs_out);
}

}  // extern "C"
