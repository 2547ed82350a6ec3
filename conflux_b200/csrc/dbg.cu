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
    DevBuf out;
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
    if (M <= 0 || N <= 0 || K <= 0 || !AT || !B || !C || at_rows <= 0 || b_rows <= 0 || c_rows <= 0 || ldat <= 0 ||
        ldb <= 0 || ldc <= 0 || at_off < 0 || b_off < 0 || row_off < 0 || col_off < 0)
        return CFLX_ERR_ARG;
    // every element the kernel may touch lies inside the buffers: AT rows of round_up(M, 2) (the producer's even copy
    // width), B rows of N, the C window; 16-byte alignment of every operand row needs even offsets
    if ((at_off & 1) || (b_off & 1) || (col_off & 1) || at_off + (K - 1) * ldat + round_up(M, 2) > (int64_t)at_rows * ldat ||
        b_off + (K - 1) * ldb + N > (int64_t)b_rows * ldb || row_off + M > c_rows || col_off + N > ldc) {
        set_last_error("dbg_gemm_tn: window outside the buffers or misaligned");
        return CFLX_ERR_ARG;
    }
    const size_t a_n = (size_t)at_rows * ldat, b_n = (size_t)b_rows * ldb, c_n = (size_t)c_rows * ldc;
    DevBuf dA, dB, dC, dC0, dD;
    CFLX_TRY(dA.alloc(sizeof(double) * a_n));
    CFLX_TRY(dB.alloc(sizeof(double) * b_n));
    CFLX_TRY(dC.alloc(sizeof(double) * c_n));
    CFLX_TRY(dC0.alloc(sizeof(double) * c_n));
    CFLX_TRY(dD.alloc(sizeof(double) * c_n));
    CFLX_CUDA(cudaMemcpy(dA.p, AT, sizeof(double) * a_n, cudaMemcpyHostToDevice));
    CFLX_CUDA(cudaMemcpy(dB.p, B, sizeof(double) * b_n, cudaMemcpyHostToDevice));
    CFLX_CUDA(cudaMemcpy(dC0.p, C, sizeof(double) * c_n, cudaMemcpyHostToDevice));
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
    if (D_out) CFLX_CUDA(cudaMemcpy(D_out, in_place ? dC.p : dD.p, sizeof(double) * c_n, cudaMemcpyDeviceToHost));
    if (C_out) CFLX_CUDA(cudaMemcpy(C_out, dC.p, sizeof(double) * c_n, cudaMemcpyDeviceToHost));
    CFLX_CUDA(cudaDeviceSynchronize());
    return CFLX_OK;
}

// D = beta*C + alpha * A * B on the narrow GEMM of the solve (solve.cu); A [M x K], B [K x N], C / D [M x N] dense
// row-major.  D == C (the same host array) runs the kernel with D aliasing C on the device.  The timed repetitions run
// first, into a separate output, and the result is one more launch on the pristine inputs.
int cflx_dbg_gemm_narrow(int M, int N, int K, const double* A, const double* B, const double* C, double alpha, double beta,
                         double* D, int reps, double* ms_out) {
    CFLX_TRY(check_device());
    if (M <= 0 || N <= 0 || K < 0 || (K & 3) || !A || !B) return CFLX_ERR_ARG;
    const size_t a_n = (size_t)M * K, b_n = (size_t)K * N, c_n = (size_t)M * N;
    DevBuf dA, dB, dC, dT;
    CFLX_TRY(dA.alloc(sizeof(double) * a_n));
    CFLX_TRY(dB.alloc(sizeof(double) * b_n));
    CFLX_TRY(dC.alloc(sizeof(double) * c_n));
    CFLX_TRY(dT.alloc(sizeof(double) * c_n));
    CFLX_CUDA(cudaMemcpy(dA.p, A, sizeof(double) * a_n, cudaMemcpyHostToDevice));
    CFLX_CUDA(cudaMemcpy(dB.p, B, sizeof(double) * b_n, cudaMemcpyHostToDevice));
    if (C) CFLX_CUDA(cudaMemcpy(dC.p, C, sizeof(double) * c_n, cudaMemcpyHostToDevice));
    else CFLX_CUDA(cudaMemset(dC.p, 0, sizeof(double) * c_n));
    const bool alias = C && D == C;
    auto run = [&](double* out) {
        return launch_gemm_narrow(M, N, K, dA.as<double>(), K, dB.as<double>(), N, dC.as<double>(), N, out, N, alpha, beta, 0);
    };
    CFLX_TRY(time_reps([&] { return run(dT.as<double>()); }, reps, ms_out));
    double* out = alias ? dC.as<double>() : dT.as<double>();
    CFLX_TRY(run(out));
    if (D) CFLX_CUDA(cudaMemcpy(D, out, sizeof(double) * c_n, cudaMemcpyDeviceToHost));
    CFLX_CUDA(cudaDeviceSynchronize());
    return CFLX_OK;
}

// D = beta*C + alpha * AT^T * B on the transposed narrow GEMM (solve.cu), like cflx_dbg_gemm_narrow; AT [K x M] is stored
// on the device with the even leading dimension round_up(M, 2), the kernel's condition, so odd M can be run.
int cflx_dbg_gemm_narrow_tn(int M, int N, int K, const double* AT, const double* B, const double* C, double alpha,
                            double beta, double* D, int reps, double* ms_out) {
    CFLX_TRY(check_device());
    if (M <= 0 || N <= 0 || K < 0 || !AT || !B) return CFLX_ERR_ARG;
    const int64_t ldat = round_up(M, 2);
    const size_t a_n = (size_t)K * ldat, b_n = (size_t)K * N, c_n = (size_t)M * N;
    DevBuf dA, dB, dC, dT;
    CFLX_TRY(dA.alloc(sizeof(double) * a_n));
    CFLX_TRY(dB.alloc(sizeof(double) * b_n));
    CFLX_TRY(dC.alloc(sizeof(double) * c_n));
    CFLX_TRY(dT.alloc(sizeof(double) * c_n));
    if (K > 0) {
        CFLX_CUDA(cudaMemcpy2D(dA.p, ldat * 8, AT, (size_t)M * 8, (size_t)M * 8, K, cudaMemcpyHostToDevice));
        CFLX_CUDA(cudaMemcpy(dB.p, B, sizeof(double) * b_n, cudaMemcpyHostToDevice));
    }
    if (C) CFLX_CUDA(cudaMemcpy(dC.p, C, sizeof(double) * c_n, cudaMemcpyHostToDevice));
    else CFLX_CUDA(cudaMemset(dC.p, 0, sizeof(double) * c_n));
    const bool alias = C && D == C;
    auto run = [&](double* out) {
        return launch_gemm_narrow_tn(M, N, K, dA.as<double>(), ldat, dB.as<double>(), N, dC.as<double>(), N, out, N, alpha,
                                     beta, 0);
    };
    CFLX_TRY(time_reps([&] { return run(dT.as<double>()); }, reps, ms_out));
    double* out = alias ? dC.as<double>() : dT.as<double>();
    CFLX_TRY(run(out));
    if (D) CFLX_CUDA(cudaMemcpy(D, out, sizeof(double) * c_n, cudaMemcpyDeviceToHost));
    CFLX_CUDA(cudaDeviceSynchronize());
    return CFLX_OK;
}

// the per-share kernels of equilibration and of the pivot growth (equil.cu) on one layer-0 share at grid position
// (pi, pj) of Px x Py; each output may be null
int cflx_dbg_equil(int Ml, int Nl, int v, int Kappa, int Px, int Py, int pi, int pj, int M, const double* A,
                   const double* r, const double* c, char equed, int ncols, double* rowmax_out, double* colmax_out,
                   double* diag_out, double* scaled_out, double* sym_scaled_out, double* growth_out, int* zero_pivot_out) {
    CFLX_TRY(check_device());
    if (Ml < 0 || Nl < 0 || v < 1 || Ml % v || Nl % v || Px < 1 || Py < 1 || pi < 0 || pi >= Px || pj < 0 || pj >= Py ||
        !A || !r || !c || M < (Ml / v) * Px * v || M < (Nl / v) * Py * v ||
        (equed != 'N' && equed != 'R' && equed != 'C' && equed != 'B'))
        return CFLX_ERR_ARG;
    const size_t a_n = (size_t)Ml * Nl;
    DevBuf dA, dW, dr, dc, dv, dg, dz;
    CFLX_TRY(dA.alloc(sizeof(double) * a_n));
    CFLX_TRY(dW.alloc(sizeof(double) * a_n));
    CFLX_TRY(dr.alloc(sizeof(double) * M));
    CFLX_TRY(dc.alloc(sizeof(double) * M));
    CFLX_TRY(dv.alloc(sizeof(double) * M));
    CFLX_TRY(dg.alloc(sizeof(double) * 2 * M));
    CFLX_TRY(dz.alloc(sizeof(int)));
    CFLX_CUDA(cudaMemcpy(dA.p, A, sizeof(double) * a_n, cudaMemcpyHostToDevice));
    CFLX_CUDA(cudaMemcpy(dr.p, r, sizeof(double) * M, cudaMemcpyHostToDevice));
    CFLX_CUDA(cudaMemcpy(dc.p, c, sizeof(double) * M, cudaMemcpyHostToDevice));
    const double* a = dA.as<double>();
    double *w = dW.as<double>(), *vec = dv.as<double>();
    const Layout L{M, v, Kappa, Ml, Nl, Px, Py, pi, pj};
    auto vec_out = [&](double* out) -> int {
        CFLX_CUDA(cudaMemcpy(out, vec, sizeof(double) * M, cudaMemcpyDeviceToHost));
        return CFLX_OK;
    };
    if (rowmax_out) {
        CFLX_TRY(equil_row_max(a, L, vec, 0));
        CFLX_TRY(vec_out(rowmax_out));
    }
    if (colmax_out) {
        CFLX_TRY(equil_col_max(a, L, dr.as<double>(), vec, 0));
        CFLX_TRY(vec_out(colmax_out));
    }
    if (diag_out) {
        CFLX_TRY(equil_diag(a, L, vec, 0));
        CFLX_TRY(vec_out(diag_out));
    }
    if (scaled_out) {
        CFLX_CUDA(cudaMemcpy(w, a, sizeof(double) * a_n, cudaMemcpyDeviceToDevice));
        CFLX_TRY(equil_apply(w, L, dr.as<double>(), dc.as<double>(), equed, 0));
        CFLX_CUDA(cudaMemcpy(scaled_out, w, sizeof(double) * a_n, cudaMemcpyDeviceToHost));
    }
    if (sym_scaled_out) {  // s = r
        CFLX_CUDA(cudaMemcpy(w, a, sizeof(double) * a_n, cudaMemcpyDeviceToDevice));
        CFLX_TRY(equil_sym_apply(w, L, dr.as<double>(), 0));
        CFLX_CUDA(cudaMemcpy(sym_scaled_out, w, sizeof(double) * a_n, cudaMemcpyDeviceToHost));
    }
    if (growth_out) {  // the share is both L\U and the input; dgesvx's maxima are those of the columns' maxima
        CFLX_TRY(equil_growth_cols(a, a, L, false, ncols, dg.as<double>(), 0));
        std::vector<double> h(2 * (size_t)M);
        CFLX_CUDA(cudaMemcpy(h.data(), dg.p, sizeof(double) * 2 * M, cudaMemcpyDeviceToHost));
        growth_out[0] = *std::max_element(h.begin() + M, h.end());
        growth_out[1] = *std::max_element(h.begin(), h.begin() + M);
    }
    if (zero_pivot_out) {
        CFLX_TRY(equil_zero_pivot(a, L, dz.as<int>(), 0));
        int z = 0;
        CFLX_CUDA(cudaMemcpy(&z, dz.p, sizeof(int), cudaMemcpyDeviceToHost));
        *zero_pivot_out = z == INT_MAX ? 0 : z;
    }
    CFLX_CUDA(cudaDeviceSynchronize());
    return CFLX_OK;
}

// the per-column pivot growth pass (equil.cu) on one layer-0 share F (the factor) and A (the input) at grid position
// (pi, pj) of Px x Py; mode 0 LU, 1 Cholesky; either output may be null
int cflx_dbg_growth_cols(int mode, int Ml, int Nl, int v, int Kappa, int Px, int Py, int pi, int pj, int M, int ncols,
                         const double* F, const double* A, double* amax_out, double* fmax_out) {
    CFLX_TRY(check_device());
    if ((mode != 0 && mode != 1) || Ml < 0 || Nl < 0 || v < 1 || Ml % v || Nl % v || Px < 1 || Py < 1 || pi < 0 ||
        pi >= Px || pj < 0 || pj >= Py || !F || !A || M < (Ml / v) * Px * v || M < (Nl / v) * Py * v)
        return CFLX_ERR_ARG;
    const size_t a_n = (size_t)Ml * Nl;
    DevBuf dF, dA, dg;
    CFLX_TRY(dF.alloc(sizeof(double) * a_n));
    CFLX_TRY(dA.alloc(sizeof(double) * a_n));
    CFLX_TRY(dg.alloc(sizeof(double) * 2 * M));
    CFLX_CUDA(cudaMemcpy(dF.p, F, sizeof(double) * a_n, cudaMemcpyHostToDevice));
    CFLX_CUDA(cudaMemcpy(dA.p, A, sizeof(double) * a_n, cudaMemcpyHostToDevice));
    const Layout L{M, v, Kappa, Ml, Nl, Px, Py, pi, pj};
    CFLX_TRY(equil_growth_cols(dF.as<double>(), dA.as<double>(), L, mode == 1, ncols, dg.as<double>(), 0));
    if (amax_out) CFLX_CUDA(cudaMemcpy(amax_out, dg.p, sizeof(double) * M, cudaMemcpyDeviceToHost));
    if (fmax_out) CFLX_CUDA(cudaMemcpy(fmax_out, dg.as<double>() + M, sizeof(double) * M, cudaMemcpyDeviceToHost));
    CFLX_CUDA(cudaDeviceSynchronize());
    return CFLX_OK;
}

// the seed, scatter and zero-fill kernels of the inverse (inverse.cu) on one share at grid position (pi, pj) of Px x Py
int cflx_dbg_inverse_share(int mode, int Ml, int Nl, int v, int Kappa, int Px, int Py, int pi, int pj, int M, int c0,
                           int nc, int rows, const double* X, int ldx, const int* perm, double* W_out,
                           double* share_inout, int zero_fill) {
    CFLX_TRY(check_device());
    if ((mode != 0 && mode != 1) || Ml < 0 || Nl < 0 || v < 1 || Ml % v || Nl % v || Px < 1 || Py < 1 || pi < 0 ||
        pi >= Px || pj < 0 || pj >= Py || M < (Ml / v) * Px * v || M < (Nl / v) * Py * v || c0 < 0 || nc < 1 ||
        c0 + nc > M || rows < 0 || rows > Ml || (share_inout && (!X || ldx < nc || (mode == 0 && !perm))))
        return CFLX_ERR_ARG;
    const Layout L{M, v, Kappa, Ml, Nl, Px, Py, pi, pj};
    const int ldn = (int)round_up(nc, 8);
    if (W_out) {
        DevBuf dW;
        CFLX_TRY(dW.alloc(sizeof(double) * Ml * ldn));
        CFLX_CUDA(cudaMemset(dW.p, 0, sizeof(double) * Ml * ldn));
        CFLX_TRY(launch_inverse_seed(dW.as<double>(), ldn, L, rows, c0, nc, 0));
        CFLX_CUDA(cudaMemcpy(W_out, dW.p, sizeof(double) * Ml * ldn, cudaMemcpyDeviceToHost));
    }
    if (share_inout) {
        const size_t a_n = (size_t)Ml * Nl;
        DevBuf dA, dX, dp;
        CFLX_TRY(dA.alloc(sizeof(double) * a_n));
        CFLX_TRY(dX.alloc(sizeof(double) * M * ldx));
        CFLX_TRY(dp.alloc(sizeof(int) * M));
        CFLX_CUDA(cudaMemcpy(dA.p, share_inout, sizeof(double) * a_n, cudaMemcpyHostToDevice));
        CFLX_CUDA(cudaMemcpy(dX.p, X, sizeof(double) * M * ldx, cudaMemcpyHostToDevice));
        if (mode == 0) CFLX_CUDA(cudaMemcpy(dp.p, perm, sizeof(int) * M, cudaMemcpyHostToDevice));
        CFLX_TRY(launch_inverse_scatter(mode == 0 ? InvKind::LU : InvKind::Chol, dX.as<double>(), ldx, c0, nc,
                                        mode == 0 ? dp.as<int>() : nullptr, L, dA.as<double>(), 0));
        if (mode == 1 && zero_fill) CFLX_TRY(launch_inverse_zero(L, dA.as<double>(), 0));
        CFLX_CUDA(cudaMemcpy(share_inout, dA.p, sizeof(double) * a_n, cudaMemcpyDeviceToHost));
    }
    CFLX_CUDA(cudaDeviceSynchronize());
    return CFLX_OK;
}

// the pack and scatter kernels of the distributed solves (solve_local.cu) on one share at grid position (pi, pj) of Px x Py
int cflx_dbg_solve_local_share(int mode, int Ml, int v, int Kappa, int Px, int Py, int pi, int pj, int M, int nrhs, int c0,
                               int w, const double* B, int ldb, double* Bk_out, const double* Xk, double* X_inout, int ldx) {
    CFLX_TRY(check_device());
    if ((mode != 0 && mode != 1) || Ml < 0 || v < 1 || Ml % v || Px < 1 || Py < 1 || pi < 0 || pi >= Px || pj < 0 ||
        pj >= Py || M < (Ml / v) * Px * v || nrhs < 1 || c0 < 0 || w < 1 || c0 + w > nrhs)
        return CFLX_ERR_ARG;
    const int ncl = rhs_local_cols(nrhs, v, Py), ldn = (int)round_up(w, 8);
    if ((Bk_out && (!B || ldb < ncl)) || (X_inout && (!Xk || ldx < ncl))) return CFLX_ERR_ARG;
    const Layout L{M, v, Kappa, Ml, ncl, Px, Py, pi, pj};
    const int rows = solve_local_rows(L, mode == 1);
    if (Bk_out) {
        DevBuf dB, dK;
        CFLX_TRY(dB.alloc(sizeof(double) * Ml * ldb));
        CFLX_TRY(dK.alloc(sizeof(double) * M * ldn));
        CFLX_CUDA(cudaMemcpy(dB.p, B, sizeof(double) * Ml * ldb, cudaMemcpyHostToDevice));
        CFLX_TRY(launch_solve_local_pack(dB.as<double>(), ldb, L, rows, c0, w, dK.as<double>(), ldn, 0));
        CFLX_CUDA(cudaMemcpy(Bk_out, dK.p, sizeof(double) * M * ldn, cudaMemcpyDeviceToHost));
    }
    if (X_inout) {
        DevBuf dX, dK;
        CFLX_TRY(dX.alloc(sizeof(double) * Ml * ldx));
        CFLX_TRY(dK.alloc(sizeof(double) * M * ldn));
        CFLX_CUDA(cudaMemcpy(dX.p, X_inout, sizeof(double) * Ml * ldx, cudaMemcpyHostToDevice));
        CFLX_CUDA(cudaMemcpy(dK.p, Xk, sizeof(double) * M * ldn, cudaMemcpyHostToDevice));
        CFLX_TRY(launch_solve_local_scatter(dK.as<double>(), ldn, L, rows, c0, w, dX.as<double>(), ldx, 0));
        CFLX_CUDA(cudaMemcpy(X_inout, dX.p, sizeof(double) * Ml * ldx, cudaMemcpyDeviceToHost));
    }
    CFLX_CUDA(cudaDeviceSynchronize());
    return CFLX_OK;
}

// the per-share passes of the 1-norm and the infinity-norm (norm.cu) on one layer-0 share at grid position (pi, pj) of
// Px x Py: mode 0 the column sums, 1 the column sums of the symmetric matrix stored as its lower triangle, 2 the row sums
int cflx_dbg_norm_share(int mode, int Ml, int Nl, int v, int Kappa, int Px, int Py, int pi, int pj, int M, const double* A,
                        double* out) {
    CFLX_TRY(check_device());
    if (mode < 0 || mode > 2 || Ml < 1 || Nl < 1 || v < 1 || Ml % v || Nl % v || Px < 1 || Py < 1 || pi < 0 || pi >= Px ||
        pj < 0 || pj >= Py || !A || !out || M < (Ml / v) * Px * v || M < (Nl / v) * Py * v)
        return CFLX_ERR_ARG;
    const Layout L{M, v, Kappa, Ml, Nl, Px, Py, pi, pj};
    const size_t a_n = (size_t)Ml * Nl;
    int ncp = 0, nrp = 0;
    norm1_partials(L, &ncp, &nrp);
    DevBuf dA, dcol, drow, dout;
    CFLX_TRY(dA.alloc(sizeof(double) * a_n));
    CFLX_TRY(dcol.alloc(sizeof(double) * ncp * Nl));
    CFLX_TRY(drow.alloc(sizeof(double) * nrp * Ml));
    CFLX_TRY(dout.alloc(sizeof(double) * M));
    CFLX_CUDA(cudaMemcpy(dA.p, A, sizeof(double) * a_n, cudaMemcpyHostToDevice));
    double* o = dout.as<double>();
    if (mode == 2) {  // norminf_grid zeroes the vector; the column sums write every entry (NaN shows one they miss)
        CFLX_CUDA(cudaMemset(o, 0, sizeof(double) * M));
        CFLX_TRY(launch_norminf_share(dA.as<double>(), L, o, 0));
    } else {
        CFLX_TRY(launch_fill(o, M, std::numeric_limits<double>::quiet_NaN(), 0));
        CFLX_TRY(launch_norm1_share(dA.as<double>(), L, mode == 1, dcol.as<double>(), drow.as<double>(), o, 0));
    }
    CFLX_CUDA(cudaMemcpy(out, o, sizeof(double) * M, cudaMemcpyDeviceToHost));
    CFLX_CUDA(cudaDeviceSynchronize());
    return CFLX_OK;
}

// cflx_chol_validate's per-share kernels on one layer-0 share at grid position (pi, pj) of Px x Py (each output may be
// null): the sum of squares of its lower triangle of the real tiles, and the masked transposed panel of step t
int cflx_dbg_chol_validate_share(int Ml, int Nl, int v, int Kappa, int Px, int Py, int pi, int pj, const double* A, int t,
                                 double* PT_out, double* sumsq_out) {
    CFLX_TRY(check_device());
    if (Ml < 1 || Nl < 1 || v < 1 || Ml % v || Nl % v || Kappa < 1 || Px < 1 || Py < 1 || pi < 0 || pi >= Px || pj < 0 ||
        pj >= Py || !A || t < 0 || t >= Kappa || (t / Py + 1) * v > Nl)
        return CFLX_ERR_ARG;
    const int M = std::max((Ml / v) * Px, (Nl / v) * Py) * v;
    const Layout L{M, v, Kappa, Ml, Nl, Px, Py, pi, pj};
    const size_t a_n = (size_t)Ml * Nl;
    const int64_t ldp = chol_panel_ld(Ml);
    DevBuf dA, dacc, dPT;
    CFLX_TRY(dA.alloc(sizeof(double) * a_n));
    CFLX_TRY(dacc.alloc(sizeof(double) * (1 + SUMSQ_PARTIALS)));
    CFLX_TRY(dPT.alloc(sizeof(double) * v * ldp));
    CFLX_CUDA(cudaMemcpy(dA.p, A, sizeof(double) * a_n, cudaMemcpyHostToDevice));
    if (sumsq_out) {
        double* acc = dacc.as<double>();
        CFLX_CUDA(cudaMemset(acc, 0, sizeof(double)));
        CFLX_TRY(launch_sumsq_lower(dA.as<double>(), L, acc + 1, acc, 0));
        CFLX_CUDA(cudaMemcpy(sumsq_out, acc, sizeof(double), cudaMemcpyDeviceToHost));
    }
    if (PT_out) {  // v x chol_panel_ld(Ml); NaN where the kernel writes nothing (and everywhere off grid column t % Py)
        CFLX_TRY(launch_fill(dPT.as<double>(), v * ldp, std::numeric_limits<double>::quiet_NaN(), 0));
        const int row0 = first_local_tile(t, pi, Px) * v;
        if (pj == t % Py)  // the guard and the arguments of cflx_chol_validate
            CFLX_TRY(launch_extract_l_panel_T(dA.as<double>(), Nl, row0, (t / Py) * v, Ml - row0, L, t, dPT.as<double>(),
                                              chol_piece_ld(L, t, pi), 0));
        CFLX_CUDA(cudaMemcpy(PT_out, dPT.p, sizeof(double) * v * ldp, cudaMemcpyDeviceToHost));
    }
    CFLX_CUDA(cudaDeviceSynchronize());
    return CFLX_OK;
}

// the two extract kernels of cflx_lu_validate's sweep, step t, on one layer-0 share C of the packed factors at grid
// position (pi, pj) of Px x Py, under the owner guards of the sweep (each output may be null)
int cflx_dbg_lu_validate_share(int Ml, int Nl, int v, int Px, int Py, int pi, int pj, const double* C, int t, double* LT_out,
                               double* U_out) {
    CFLX_TRY(check_device());
    if (Ml < 1 || Nl < 1 || v < 1 || Ml % v || Nl % v || Px < 1 || Py < 1 || pi < 0 || pi >= Px || pj < 0 || pj >= Py ||
        !C || t < 0 || (Ml / v) * Px != (Nl / v) * Py)  // the LU's shares of an M x M matrix
        return CFLX_ERR_ARG;
    const int M = (Ml / v) * Px * v;
    if (t >= M / v) return CFLX_ERR_ARG;
    const Layout L{M, v, M / v, Ml, Nl, Px, Py, pi, pj};
    const size_t a_n = (size_t)Ml * Nl;
    const int64_t ldp = round_up(Ml, 2);
    const double nan = std::numeric_limits<double>::quiet_NaN();
    DevBuf dC, dLT, dU;
    CFLX_TRY(dC.alloc(sizeof(double) * a_n));
    CFLX_TRY(dLT.alloc(sizeof(double) * v * ldp));
    CFLX_TRY(dU.alloc(sizeof(double) * v * Nl));
    CFLX_CUDA(cudaMemcpy(dC.p, C, sizeof(double) * a_n, cudaMemcpyHostToDevice));
    if (LT_out) {  // v x round_up(Ml, 2), NaN where the kernel writes nothing
        CFLX_TRY(launch_fill(dLT.as<double>(), v * ldp, nan, 0));
        CFLX_TRY(launch_lu_extract_l(dC.as<double>(), L, t, dLT.as<double>(), ldp, 0));
        CFLX_CUDA(cudaMemcpy(LT_out, dLT.p, sizeof(double) * v * ldp, cudaMemcpyDeviceToHost));
    }
    if (U_out) {  // v x Nl
        CFLX_TRY(launch_fill(dU.as<double>(), (int64_t)v * Nl, nan, 0));
        CFLX_TRY(launch_lu_extract_u(dC.as<double>(), L, t, dU.as<double>(), Nl, 0));
        CFLX_CUDA(cudaMemcpy(U_out, dU.p, sizeof(double) * v * Nl, cudaMemcpyDeviceToHost));
    }
    CFLX_CUDA(cudaDeviceSynchronize());
    return CFLX_OK;
}

// the Cholesky update's column-operand gather (chol.cu) on one share of Ml x Nl at grid column pj of Px x Py, from the
// Px broadcast pieces of the panel of global tiles >= gfirst (host: piece p is v x chol_piece_ld(p), back to back), for
// the local column tiles with global index >= gfirst (Bc's tile t: local tile lj0 + t); Bc_out is v x Nl, NaN where
// nothing is written
int cflx_dbg_chol_gather_cols(int v, int Px, int Py, int pj, int Ml, int Nl, int gfirst, const double* pieces,
                              double* Bc_out) {
    CFLX_TRY(check_device());
    if (v < 1 || Px < 1 || Py < 1 || pj < 0 || pj >= Py || Ml < 1 || Nl < 1 || Ml % v || Nl % v || gfirst < 0 || !pieces ||
        !Bc_out)
        return CFLX_ERR_ARG;
    const Layout L{0, v, 0, Ml, Nl, Px, Py, 0, pj};  // chol_piece_ld reads Ml, v and Px only
    const int64_t ldp = chol_panel_ld(Ml), piece_stride = (int64_t)v * ldp, ldb = Nl;
    const double nan = std::numeric_limits<double>::quiet_NaN();
    DevBuf dG, dB;
    CFLX_TRY(dG.alloc(sizeof(double) * Px * piece_stride));
    CFLX_TRY(dB.alloc(sizeof(double) * v * ldb));
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
            set_last_error("dbg_chol_gather_cols: column tile %d reads outside the pieces", j);
            return CFLX_ERR_ARG;
        }
    }
    if (ntc > 0)
        CFLX_TRY(launch_gather_cols(dG.as<double>(), piece_stride, dB.as<double>(), ldb, v, Px, Py, pj, lj0, ntc, gfirst, Ml, 0));
    CFLX_CUDA(cudaMemcpy(Bc_out, dB.p, sizeof(double) * v * ldb, cudaMemcpyDeviceToHost));
    CFLX_CUDA(cudaDeviceSynchronize());
    return CFLX_OK;
}

// the refinement's assembly (refine.cu) from the host chunks of Px Py Pz ranks: mode 0 dgerfs' R, ratio and W; 1
// dla_lin_berr's R, ratio and Q; 2 the double-double R.  safe1, safe2 and nz eps are refine_safe's for M.
int cflx_dbg_refine_assemble(int mode, int Px, int Py, int Pz, int v, int M, int Ml, int Nl, int nn, int tn, int nrhs,
                             int ldn, const double* all, const double* B, double* R_out, double* ratio_out, double* W_out,
                             double* Q_out) {
    CFLX_TRY(check_device());
    if (mode < 0 || mode > 2 || Px < 1 || Py < 1 || Pz < 1 || v < 1 || M < 1 || Ml < 0 || Nl < 0 || Ml % v || Nl % v ||
        (!nn && !tn) || nrhs < 1 || ldn < nrhs || !all || !B || (nn && M > (Ml / v) * Px * v) ||
        (tn && M > (Nl / v) * Py * v))
        return CFLX_ERR_ARG;
    const int64_t chunk = (int64_t)((nn ? Ml : 0) + (tn ? Nl : 0)) * 2 * ldn, mat = (int64_t)M * ldn;
    const int64_t all_n = chunk * Px * Py * Pz;
    DevBuf dall, dB, dR, dratio, dW, dQ;
    CFLX_TRY(dall.alloc(sizeof(double) * all_n));
    for (DevBuf* b : {&dB, &dR, &dratio, &dW, &dQ}) CFLX_TRY(b->alloc(sizeof(double) * mat));
    CFLX_CUDA(cudaMemcpy(dall.p, all, sizeof(double) * all_n, cudaMemcpyHostToDevice));
    CFLX_CUDA(cudaMemcpy(dB.p, B, sizeof(double) * mat, cudaMemcpyHostToDevice));
    const double nan = std::numeric_limits<double>::quiet_NaN();
    for (DevBuf* b : {&dR, &dratio, &dW, &dQ}) CFLX_TRY(launch_fill(b->as<double>(), mat, nan, 0));
    double safe1, safe2, nzeps;
    refine_safe(M, &safe1, &safe2, &nzeps);
    AssembleArgs a{dall.as<double>(), chunk, Ml, Nl, ldn, nrhs, M, nn != 0, tn != 0, v, Px, Py, Pz, dB.as<double>(),
                   dR.as<double>(), dratio.as<double>(), mode == 1 ? nullptr : dW.as<double>(), safe1, safe2, nzeps};
    a.lin_berr = mode == 1;
    a.Q = mode == 1 ? dQ.as<double>() : nullptr;
    CFLX_TRY(launch_assemble(a, mode == 2, 0));
    auto out = [&](double* h, DevBuf& d) -> int {
        if (h) CFLX_CUDA(cudaMemcpy(h, d.p, sizeof(double) * mat, cudaMemcpyDeviceToHost));
        return CFLX_OK;
    };
    CFLX_TRY(out(R_out, dR));
    CFLX_TRY(out(ratio_out, dratio));
    CFLX_TRY(out(W_out, dW));
    CFLX_TRY(out(Q_out, dQ));
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
    if (M < 1 || nrhs < 1 || ldn < nrhs || !A || ((stats_out || add_out || Y_out) && !D) ||
        ((select_out || add_out || Y_out) && !sel) || (!Y_out != !T_inout))
        return CFLX_ERR_ARG;
    const int64_t mat = (int64_t)M * ldn;
    DevBuf dA, dD, dd, dsel, dW, dT, dv;
    CFLX_TRY(dA.alloc(sizeof(double) * mat));
    CFLX_TRY(dD.alloc(sizeof(double) * mat));
    CFLX_TRY(dd.alloc(sizeof(double) * M));
    CFLX_TRY(dsel.alloc(sizeof(int) * ldn));
    CFLX_TRY(dW.alloc(sizeof(double) * mat));
    CFLX_TRY(dT.alloc(sizeof(double) * mat));
    CFLX_TRY(dv.alloc(sizeof(double) * nrhs * REFINE_NSTAT));
    CFLX_CUDA(cudaMemcpy(dA.p, A, sizeof(double) * mat, cudaMemcpyHostToDevice));
    if (D) CFLX_CUDA(cudaMemcpy(dD.p, D, sizeof(double) * mat, cudaMemcpyHostToDevice));
    if (d) CFLX_CUDA(cudaMemcpy(dd.p, d, sizeof(double) * M, cudaMemcpyHostToDevice));
    if (sel) CFLX_CUDA(cudaMemcpy(dsel.p, sel, sizeof(int) * ldn, cudaMemcpyHostToDevice));
    const double* a = dA.as<double>();
    double* w = dW.as<double>();
    if (max_out) {
        CFLX_TRY(launch_column_max(a, M, ldn, nrhs, dv.as<double>(), 0));
        CFLX_CUDA(cudaMemcpy(max_out, dv.p, sizeof(double) * nrhs, cudaMemcpyDeviceToHost));
    }
    if (stats_out) {
        CFLX_TRY(launch_column_stats(a, dD.as<double>(), d ? dd.as<double>() : nullptr, M, ldn, nrhs, dv.as<double>(), 0));
        CFLX_CUDA(cudaMemcpy(stats_out, dv.p, sizeof(double) * nrhs * REFINE_NSTAT, cudaMemcpyDeviceToHost));
    }
    if (select_out) {
        CFLX_TRY(launch_fill(w, mat, std::numeric_limits<double>::quiet_NaN(), 0));
        CFLX_TRY(launch_select_cols(a, dsel.as<int>(), M, ldn, w, 0));
        CFLX_CUDA(cudaMemcpy(select_out, w, sizeof(double) * mat, cudaMemcpyDeviceToHost));
    }
    if (add_out) {
        CFLX_CUDA(cudaMemcpy(w, a, sizeof(double) * mat, cudaMemcpyDeviceToDevice));
        CFLX_TRY(launch_add_cols(w, dD.as<double>(), dsel.as<int>(), M, ldn, 0));
        CFLX_CUDA(cudaMemcpy(add_out, w, sizeof(double) * mat, cudaMemcpyDeviceToHost));
    }
    if (Y_out) {
        CFLX_CUDA(cudaMemcpy(w, a, sizeof(double) * mat, cudaMemcpyDeviceToDevice));
        CFLX_CUDA(cudaMemcpy(dT.p, T_inout, sizeof(double) * mat, cudaMemcpyHostToDevice));
        CFLX_TRY(launch_update_x(w, dT.as<double>(), dD.as<double>(), dsel.as<int>(), M, ldn, 0));
        CFLX_CUDA(cudaMemcpy(Y_out, w, sizeof(double) * mat, cudaMemcpyDeviceToHost));
        CFLX_CUDA(cudaMemcpy(T_inout, dT.p, sizeof(double) * mat, cudaMemcpyDeviceToHost));
    }
    CFLX_CUDA(cudaDeviceSynchronize());
    return CFLX_OK;
}

// the determinant's product kernel (det.cu) on host vectors
int cflx_dbg_det(int n, const double* d, const double* s1, const double* s2, int square, double* mant_out,
                 int64_t* exp_out, int* neg_out, int* first_zero_out, int* nonfinite_out) {
    CFLX_TRY(check_device());
    if (n < 1 || !d || (square != 0 && square != 1)) return CFLX_ERR_ARG;
    DevBuf dv, dr;
    CFLX_TRY(dv.alloc(sizeof(double) * 3 * (size_t)n));
    CFLX_TRY(dr.alloc(sizeof(DetResult)));
    double* v = dv.as<double>();
    CFLX_CUDA(cudaMemcpy(v, d, sizeof(double) * n, cudaMemcpyHostToDevice));
    if (s1) CFLX_CUDA(cudaMemcpy(v + n, s1, sizeof(double) * n, cudaMemcpyHostToDevice));
    if (s2) CFLX_CUDA(cudaMemcpy(v + 2 * (size_t)n, s2, sizeof(double) * n, cudaMemcpyHostToDevice));
    CFLX_TRY(launch_det(v, s1 ? v + n : nullptr, s2 ? v + 2 * (size_t)n : nullptr, n, square != 0, dr.as<DetResult>(), 0));
    DetResult r{};
    CFLX_CUDA(cudaMemcpy(&r, dr.p, sizeof(r), cudaMemcpyDeviceToHost));
    if (mant_out) *mant_out = r.mant;
    if (exp_out) *exp_out = r.exp;
    if (neg_out) *neg_out = r.neg;
    if (first_zero_out) *first_zero_out = r.first_zero;
    if (nonfinite_out) *nonfinite_out = r.nonfinite;
    return CFLX_OK;
}

// the residual kernels of the refinement (refine.cu) on one layer-0 share; the timed repetitions run first, then the
// launch whose result is returned
int cflx_dbg_residual(int mode, int Ml, int Nl, const double* A, int v, int Kappa, int Px, int Py, int pi, int pj,
                      int nrhs, const double* Xc, const double* Xr, double* P_out, double* Q_out, int reps, double* ms_out) {
    CFLX_TRY(check_device());
    if (mode < 0 || mode > 2 || Ml < 0 || Nl < 0 || (Nl & 1) || v < 4 || (v & 3) || nrhs < 1 || !A || Px < 1 || Py < 1 ||
        pi < 0 || pi >= Px || pj < 0 || pj >= Py || (mode != 1 && !Xc) || (mode != 0 && !Xr))
        return CFLX_ERR_ARG;
    const ResidMode m = mode == 0 ? ResidMode::NN : mode == 1 ? ResidMode::TN : ResidMode::SymLower;
    const int rows = mode == 0 ? Ml : mode == 1 ? Nl : Ml + Nl;
    const size_t a_n = (size_t)Ml * Nl, o_n = (size_t)std::max(rows, 1) * nrhs;
    DevBuf dA, dXc, dXr, dP, dQ;
    CFLX_TRY(dA.alloc(sizeof(double) * a_n));
    CFLX_TRY(dXc.alloc(sizeof(double) * (size_t)Nl * nrhs));
    CFLX_TRY(dXr.alloc(sizeof(double) * (size_t)Ml * nrhs));
    CFLX_TRY(dP.alloc(sizeof(double) * o_n));
    CFLX_TRY(dQ.alloc(sizeof(double) * o_n));
    CFLX_CUDA(cudaMemcpy(dA.p, A, sizeof(double) * a_n, cudaMemcpyHostToDevice));
    if (Xc) CFLX_CUDA(cudaMemcpy(dXc.p, Xc, sizeof(double) * (size_t)Nl * nrhs, cudaMemcpyHostToDevice));
    if (Xr) CFLX_CUDA(cudaMemcpy(dXr.p, Xr, sizeof(double) * (size_t)Ml * nrhs, cudaMemcpyHostToDevice));
    const Layout L{0, v, Kappa, Ml, Nl, Px, Py, pi, pj};  // M: the kernels index by local row and column only
    auto run = [&]() {
        return launch_residual(m, dA.as<double>(), L, dXc.as<double>(), dXr.as<double>(), nrhs, nrhs, dP.as<double>(),
                               dQ.as<double>(), nrhs, 0);
    };
    CFLX_TRY(time_reps(run, reps, ms_out));
    CFLX_CUDA(cudaMemset(dP.p, 0, sizeof(double) * o_n));
    CFLX_CUDA(cudaMemset(dQ.p, 0, sizeof(double) * o_n));
    CFLX_TRY(run());
    if (P_out) CFLX_CUDA(cudaMemcpy(P_out, dP.p, sizeof(double) * (size_t)rows * nrhs, cudaMemcpyDeviceToHost));
    if (Q_out) CFLX_CUDA(cudaMemcpy(Q_out, dQ.p, sizeof(double) * (size_t)rows * nrhs, cudaMemcpyDeviceToHost));
    CFLX_CUDA(cudaDeviceSynchronize());
    return CFLX_OK;
}

int cflx_dbg_residual_x(int mode, int Ml, int Nl, const double* A, int v, int Kappa, int Px, int Py, int pi, int pj,
                        int nrhs, const double* Xc, const double* Xct, const double* Xr, const double* Xrt, double* hi_out,
                        double* lo_out, int reps, double* ms_out) {
    CFLX_TRY(check_device());
    if (mode < 0 || mode > 2 || Ml < 0 || Nl < 0 || v < 1 || nrhs < 1 || !A || Px < 1 || Py < 1 || pi < 0 || pi >= Px ||
        pj < 0 || pj >= Py || (mode != 1 && !Xc) || (mode != 0 && !Xr))
        return CFLX_ERR_ARG;
    const ResidMode m = mode == 0 ? ResidMode::NN : mode == 1 ? ResidMode::TN : ResidMode::SymLower;
    const int rows = mode == 0 ? Ml : mode == 1 ? Nl : Ml + Nl;
    const size_t a_n = (size_t)Ml * Nl, o_n = (size_t)std::max(rows, 1) * nrhs;
    const size_t c_n = (size_t)Nl * nrhs, r_n = (size_t)Ml * nrhs;
    DevBuf dA, dXc, dXct, dXr, dXrt, dH, dL;
    CFLX_TRY(dA.alloc(sizeof(double) * a_n));
    CFLX_TRY(dXc.alloc(sizeof(double) * c_n));
    CFLX_TRY(dXct.alloc(sizeof(double) * c_n));
    CFLX_TRY(dXr.alloc(sizeof(double) * r_n));
    CFLX_TRY(dXrt.alloc(sizeof(double) * r_n));
    CFLX_TRY(dH.alloc(sizeof(double) * o_n));
    CFLX_TRY(dL.alloc(sizeof(double) * o_n));
    CFLX_CUDA(cudaMemcpy(dA.p, A, sizeof(double) * a_n, cudaMemcpyHostToDevice));
    if (Xc) CFLX_CUDA(cudaMemcpy(dXc.p, Xc, sizeof(double) * c_n, cudaMemcpyHostToDevice));
    if (Xct) CFLX_CUDA(cudaMemcpy(dXct.p, Xct, sizeof(double) * c_n, cudaMemcpyHostToDevice));
    if (Xr) CFLX_CUDA(cudaMemcpy(dXr.p, Xr, sizeof(double) * r_n, cudaMemcpyHostToDevice));
    if (Xrt) CFLX_CUDA(cudaMemcpy(dXrt.p, Xrt, sizeof(double) * r_n, cudaMemcpyHostToDevice));
    const Layout L{0, v, Kappa, Ml, Nl, Px, Py, pi, pj};
    auto run = [&]() {
        return launch_residual_x(m, dA.as<double>(), L, dXc.as<double>(), Xct ? dXct.as<double>() : nullptr,
                                 dXr.as<double>(), Xrt ? dXrt.as<double>() : nullptr, nrhs, nrhs, dH.as<double>(),
                                 dL.as<double>(), nrhs, 0);
    };
    CFLX_TRY(time_reps(run, reps, ms_out));
    CFLX_CUDA(cudaMemset(dH.p, 0, sizeof(double) * o_n));
    CFLX_CUDA(cudaMemset(dL.p, 0, sizeof(double) * o_n));
    CFLX_TRY(run());
    if (hi_out) CFLX_CUDA(cudaMemcpy(hi_out, dH.p, sizeof(double) * (size_t)rows * nrhs, cudaMemcpyDeviceToHost));
    if (lo_out) CFLX_CUDA(cudaMemcpy(lo_out, dL.p, sizeof(double) * (size_t)rows * nrhs, cudaMemcpyDeviceToHost));
    CFLX_CUDA(cudaDeviceSynchronize());
    return CFLX_OK;
}

int cflx_dbg_panel(int n, int v, const double* panel, int* perm_out, double* A00_out, double* LU_out, int reps,
                   double* ms_out) {
    CFLX_TRY(check_device());
    if (n < 0 || v <= 0) return CFLX_ERR_ARG;
    const int64_t ld = std::max<int64_t>(2, round_up(n, 2));
    // host transpose into the kernel's K-major layout
    std::vector<double> WT((size_t)v * ld, 0.0);
    for (int r = 0; r < n; ++r)
        for (int c = 0; c < v; ++c) WT[(size_t)c * ld + r] = panel[(size_t)r * v + c];
    DevBuf dW, dW0, dA00, dA00T, dperm;
    CFLX_TRY(dW.alloc(sizeof(double) * v * ld));
    CFLX_TRY(dW0.alloc(sizeof(double) * v * ld));
    CFLX_TRY(dA00.alloc(sizeof(double) * v * v));
    CFLX_TRY(dA00T.alloc(sizeof(double) * v * v));
    CFLX_TRY(dperm.alloc(sizeof(int) * 2 * v));
    CFLX_CUDA(cudaMemcpy(dW0.p, WT.data(), sizeof(double) * v * ld, cudaMemcpyHostToDevice));
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
    panel_workspace_destroy(&ws);
    if (rc != CFLX_OK) {
        if (rc == CFLX_ERR_CUDA) set_last_error("panel kernel failed: %s", cudaGetErrorString(cudaGetLastError()));
        return rc;
    }
    if (ms_out) *ms_out = total / reps;
    if (perm_out) CFLX_CUDA(cudaMemcpy(perm_out, dperm.p, sizeof(int) * v, cudaMemcpyDeviceToHost));
    if (A00_out) CFLX_CUDA(cudaMemcpy(A00_out, dA00.p, sizeof(double) * v * v, cudaMemcpyDeviceToHost));
    if (LU_out) {
        CFLX_CUDA(cudaMemcpy(WT.data(), dW.p, sizeof(double) * v * ld, cudaMemcpyDeviceToHost));
        for (int r = 0; r < n; ++r)
            for (int c = 0; c < v; ++c) LU_out[(size_t)r * v + c] = WT[(size_t)c * ld + r];
    }
    CFLX_CUDA(cudaDeviceSynchronize());
    return CFLX_OK;
}

int cflx_dbg_trsm(int n, int v, int nb, int64_t ld, const double* A00, const double* B, double* X_out, const double* R,
                  double* Y_out) {
    CFLX_TRY(check_device());
    if (n <= 0 || v <= 0 || v % 4 != 0) return CFLX_ERR_ARG;
    if (nb == 0)
        for (int c : {128, 64, 32, 16, 8, 4})
            if (!nb && v % c == 0) nb = c;
    if (nb != 4 && nb != 8 && nb != 16 && nb != 32 && nb != 64 && nb != 128) return CFLX_ERR_UNSUPPORTED;
    if (v % nb != 0) return CFLX_ERR_ARG;
    if (ld == 0) ld = round_up(n, 2);
    if ((ld & 1) || ld < round_up(n, 2)) return CFLX_ERR_ARG;
    // the padding columns [n, ld) of the operand panels hold NaN: they must not reach the n solved columns
    const double nan = std::numeric_limits<double>::quiet_NaN();
    std::vector<double> A00T((size_t)v * v), BT((size_t)v * ld, nan), RT((size_t)v * ld, nan);
    for (int i = 0; i < v; ++i)
        for (int j = 0; j < v; ++j) A00T[(size_t)j * v + i] = A00[(size_t)i * v + j];
    DevBuf dA, dAT, dUinv, dLinvT, dP, dL, dR, dU;
    CFLX_TRY(dA.alloc(8 * (size_t)v * v)); CFLX_TRY(dAT.alloc(8 * (size_t)v * v));
    CFLX_TRY(dUinv.alloc(8 * (size_t)v * v)); CFLX_TRY(dLinvT.alloc(8 * (size_t)v * v));
    CFLX_TRY(dP.alloc(8 * (size_t)v * ld)); CFLX_TRY(dL.alloc(8 * (size_t)v * ld));
    CFLX_TRY(dR.alloc(8 * (size_t)v * ld)); CFLX_TRY(dU.alloc(8 * (size_t)v * ld));
    CFLX_CUDA(cudaMemcpy(dA.p, A00, 8 * (size_t)v * v, cudaMemcpyHostToDevice));
    CFLX_CUDA(cudaMemcpy(dAT.p, A00T.data(), 8 * (size_t)v * v, cudaMemcpyHostToDevice));
    CFLX_TRY(launch_diag_inverses(dA.as<double>(), v, nb, dUinv.as<double>(), dLinvT.as<double>(), 0));
    if (B && X_out) {  // X = B * U^-1, B is n x v row-major
        for (int r = 0; r < n; ++r)
            for (int c = 0; c < v; ++c) BT[(size_t)c * ld + r] = B[(size_t)r * v + c];
        CFLX_CUDA(cudaMemcpy(dP.p, BT.data(), 8 * (size_t)v * ld, cudaMemcpyHostToDevice));
        CFLX_CUDA(cudaMemset(dL.p, 0, 8 * (size_t)v * ld));
        CFLX_TRY(trsm_right_upper_T(dA.as<double>(), dUinv.as<double>(), v, nb, dP.as<double>(), dL.as<double>(), ld, n, 0));
        CFLX_CUDA(cudaMemcpy(BT.data(), dL.p, 8 * (size_t)v * ld, cudaMemcpyDeviceToHost));
        for (int r = 0; r < n; ++r)
            for (int c = 0; c < v; ++c) X_out[(size_t)r * v + c] = BT[(size_t)c * ld + r];
    }
    if (R && Y_out) {  // Y = L^-1 * R, R is v x n row-major
        for (int i = 0; i < v; ++i)
            for (int c = 0; c < n; ++c) RT[(size_t)i * ld + c] = R[(size_t)i * n + c];
        CFLX_CUDA(cudaMemcpy(dR.p, RT.data(), 8 * (size_t)v * ld, cudaMemcpyHostToDevice));
        CFLX_CUDA(cudaMemset(dU.p, 0, 8 * (size_t)v * ld));
        CFLX_TRY(trsm_left_lower_unit(dAT.as<double>(), dLinvT.as<double>(), v, nb, dR.as<double>(), dU.as<double>(), ld,
                                      (int)round_up(n, 2), 0));
        CFLX_CUDA(cudaMemcpy(RT.data(), dU.p, 8 * (size_t)v * ld, cudaMemcpyDeviceToHost));
        for (int i = 0; i < v; ++i)
            for (int c = 0; c < n; ++c) Y_out[(size_t)i * n + c] = RT[(size_t)i * ld + c];
    }
    CFLX_CUDA(cudaDeviceSynchronize());
    return CFLX_OK;
}

// inverses of the nb x nb diagonal blocks of the v x v row-major A00 = L\U: Uinv_out / LinvT_out are [v / nb][nb][nb]
int cflx_dbg_diag_inverse(int v, int nb, const double* A00, double* Uinv_out, double* LinvT_out) {
    CFLX_TRY(check_device());
    if (v <= 0 || nb <= 0 || v % nb != 0 || !A00) return CFLX_ERR_ARG;
    const size_t vv = (size_t)v * v, blocks = (size_t)v * nb;
    DevBuf dA, dU, dL;
    CFLX_TRY(dA.alloc(8 * vv));
    CFLX_TRY(dU.alloc(8 * blocks));
    CFLX_TRY(dL.alloc(8 * blocks));
    CFLX_CUDA(cudaMemcpy(dA.p, A00, 8 * vv, cudaMemcpyHostToDevice));
    CFLX_TRY(launch_diag_inverses(dA.as<double>(), v, nb, dU.as<double>(), dL.as<double>(), 0));
    if (Uinv_out) CFLX_CUDA(cudaMemcpy(Uinv_out, dU.p, 8 * blocks, cudaMemcpyDeviceToHost));
    if (LinvT_out) CFLX_CUDA(cudaMemcpy(LinvT_out, dL.p, 8 * blocks, cudaMemcpyDeviceToHost));
    CFLX_CUDA(cudaDeviceSynchronize());
    return CFLX_OK;
}

// Cholesky of one v x v row-major tile A (lower triangle read) on the kernels of the factorisation.  variant 0: the
// one-CTA potrf_tile_kernel (4 <= v <= 512); 1: potrf128_kernel (v == 128); 2: the 128-block driver potrf_tile()
// (v % 128 == 0, v >= 256).  L_out = L (zeros above the diagonal), LT_out = L^T, info_out = 1 + first failing column or 0.
int cflx_dbg_potrf_tile(int v, const double* A, double* L_out, double* LT_out, int* info_out, int variant) {
    CFLX_TRY(check_device());
    if (!A || v < 4 || v > 512 || variant < 0 || variant > 2 || (variant == 1 && v != 128) ||
        (variant == 2 && potrf_tile_scratch(v) == 0))
        return CFLX_ERR_ARG;
    const size_t vv = (size_t)v * v;
    DevBuf dD, dUT, dUc, dQ, dinfo;
    CFLX_TRY(dD.alloc(8 * vv));
    CFLX_TRY(dUT.alloc(8 * vv));
    CFLX_TRY(dUc.alloc(8 * vv));
    CFLX_TRY(dinfo.alloc(sizeof(int)));
    if (variant == 2) CFLX_TRY(dQ.alloc(8 * potrf_tile_scratch(v)));
    CFLX_CUDA(cudaMemcpy(dD.p, A, 8 * vv, cudaMemcpyHostToDevice));
    CFLX_CUDA(cudaMemset(dUT.p, 0, 8 * vv));
    CFLX_CUDA(cudaMemset(dinfo.p, 0, sizeof(int)));
    CFLX_TRY(potrf_setup(v));
    int64_t launches = 0;
    if (variant == 1)
        CFLX_TRY(potrf_block128(dD.as<double>(), v, dUT.as<double>(), v, dUc.as<double>(), dinfo.as<int>(), 0, 0));
    else
        CFLX_TRY(potrf_tile(dD.as<double>(), dUT.as<double>(), dQ.as<double>(), dinfo.as<int>(), 0, v, 0, &launches));
    if (L_out) CFLX_CUDA(cudaMemcpy(L_out, dD.p, 8 * vv, cudaMemcpyDeviceToHost));
    if (LT_out) CFLX_CUDA(cudaMemcpy(LT_out, dUT.p, 8 * vv, cudaMemcpyDeviceToHost));
    if (info_out) CFLX_CUDA(cudaMemcpy(info_out, dinfo.p, sizeof(int), cudaMemcpyDeviceToHost));
    CFLX_CUDA(cudaDeviceSynchronize());
    return CFLX_OK;
}

// step 2 of the LU loop in isolation on ONE rank (Px = 1): plan_moves (analyze_pivots) + push_phase1..3 (push_pivots_up,
// conflux_opt.hpp:176-218) + the gri/igri bookkeeping, on an n_rows x n_cols row-major matrix (n_cols even).  The npiv
// pivot rows (local indices >= fnpr, tournament order) end up in rows [fnpr, fnpr+npiv) in that order.
// gri_out[n_rows] (optional) = new row -> old row.  a01_out (optional, npiv x n_cols) = the pivot rows phase 1 extracts.
int cflx_dbg_push_pivots(int n_rows, int n_cols, double* A_inout, int npiv, const int* pivot_rows, int fnpr, int* gri_out,
                         double* a01_out) {
    CFLX_TRY(check_device());
    if (n_rows <= 0 || n_cols <= 0 || (n_cols & 1) || npiv < 0 || npiv > n_rows - fnpr || fnpr < 0) return CFLX_ERR_ARG;
    if (npiv == 0) {
        if (gri_out) for (int i = 0; i < n_rows; ++i) gri_out[i] = i;
        return CFLX_OK;
    }
    const int v = npiv;  // every pivot of the "tile" lives on this rank
    DevBuf dA, dtmp, da01, dplan, dgp, dgri, dgrit, digri;
    CFLX_TRY(dA.alloc(8 * (size_t)n_rows * n_cols));
    CFLX_TRY(dtmp.alloc(8 * (size_t)v * n_cols));
    CFLX_TRY(da01.alloc(8 * (size_t)v * n_cols));
    CFLX_TRY(dplan.alloc(sizeof(int) * (6 * (size_t)v + 8 + n_rows)));
    CFLX_TRY(dgp.alloc(sizeof(int) * v));
    CFLX_TRY(dgri.alloc(sizeof(int) * n_rows));
    CFLX_TRY(dgrit.alloc(sizeof(int) * n_rows));
    CFLX_TRY(digri.alloc(sizeof(int) * n_rows));
    CFLX_CUDA(cudaMemcpy(dA.p, A_inout, 8 * (size_t)n_rows * n_cols, cudaMemcpyHostToDevice));
    CFLX_CUDA(cudaMemcpy(dgp.p, pivot_rows, sizeof(int) * v, cudaMemcpyHostToDevice));
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
    CFLX_CUDA(cudaMemcpy(A_inout, dA.p, 8 * (size_t)n_rows * n_cols, cudaMemcpyDeviceToHost));
    if (gri_out) CFLX_CUDA(cudaMemcpy(gri_out, dgri.p, sizeof(int) * n_rows, cudaMemcpyDeviceToHost));
    if (a01_out) CFLX_CUDA(cudaMemcpy(a01_out, da01.p, 8 * (size_t)v * n_cols, cudaMemcpyDeviceToHost));
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
    if (M <= 0 || N <= 0 || K <= 0 || (N & 1) || row0 < 0 || col0 < 0 || max_ctas < 0) return CFLX_ERR_ARG;
    // AT holds row0 + M operand rows, B col0 + N columns; the planes of all of them are made (B's in the two windows
    // [0, col0) and [col0, col0 + N), as the factorisation's look-ahead splits them), the product reads the window
    const int Ma = row0 + M, Nb = col0 + N;
    const int64_t ldat = round_up(Ma, 2), ldb = Nb, ldc = N;
    DevBuf dA, dB, dC, dC0;
    CFLX_TRY(dA.alloc(sizeof(double) * K * ldat));
    CFLX_TRY(dB.alloc(sizeof(double) * K * ldb));
    CFLX_TRY(dC.alloc(sizeof(double) * M * ldc));
    CFLX_TRY(dC0.alloc(sizeof(double) * M * ldc));
    CFLX_CUDA(cudaMemset(dA.p, 0, sizeof(double) * K * ldat));
    CFLX_CUDA(cudaMemcpy2D(dA.p, ldat * 8, AT, (size_t)Ma * 8, (size_t)Ma * 8, K, cudaMemcpyHostToDevice));
    CFLX_CUDA(cudaMemcpy(dB.p, B, sizeof(double) * K * ldb, cudaMemcpyHostToDevice));
    if (C) CFLX_CUDA(cudaMemcpy(dC0.p, C, sizeof(double) * M * ldc, cudaMemcpyHostToDevice));
    else CFLX_CUDA(cudaMemset(dC0.p, 0, sizeof(double) * M * ldc));
    Events<3> ev;
    CFLX_TRY(ev.create());
    OzakiWorkspace ws;
    int rc = ozaki_workspace_create(&ws, Ma, Nb, K);
    if (reps < 1) reps = 1;
    float ms = 0, ms_split = 0;
    for (int r = 0; r < reps + 1 && rc == CFLX_OK; ++r) {
        cudaMemcpyAsync(dC.p, dC0.p, sizeof(double) * M * ldc, cudaMemcpyDeviceToDevice, 0);
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
    if (rc == CFLX_OK) {
        if (D) cudaMemcpy(D, dC.p, sizeof(double) * M * ldc, cudaMemcpyDeviceToHost);
        for (int s = 0; s < 8; ++s) {
            if (planesA_out) cudaMemcpy(planesA_out + (size_t)s * Ma * K, ws.planesA + (size_t)s * ws.cap_a * K, (size_t)Ma * K, cudaMemcpyDeviceToHost);
            if (planesB_out) cudaMemcpy(planesB_out + (size_t)s * Nb * K, ws.planesB + (size_t)s * ws.cap_b * K, (size_t)Nb * K, cudaMemcpyDeviceToHost);
        }
        if (ea_out) cudaMemcpy(ea_out, ws.ea, sizeof(int) * Ma, cudaMemcpyDeviceToHost);
        if (eb_out) cudaMemcpy(eb_out, ws.eb, sizeof(int) * Nb, cudaMemcpyDeviceToHost);
        if (cudaDeviceSynchronize() != cudaSuccess) rc = CFLX_ERR_CUDA;
    }
    ozaki_workspace_destroy(&ws);
    if (ms_out) *ms_out = ms / reps;
    if (split_ms_out) *split_ms_out = ms_split / reps;
    return rc;
}

// raw int8 tensor-core rate of back-to-back wgmma 64 x n x 32 instructions (two warpgroups per CTA, one CTA per SM,
// operands resident in shared memory).  Returns tera-MACs per second (x2 = TOP/s).
int cflx_dbg_wgmma_peak(int n, double* tmacs_out) {
    CFLX_TRY(check_device());
    if (!tmacs_out) return CFLX_ERR_ARG;
    return wgmma_peak_probe(n, tmacs_out);
}

}  // extern "C"
