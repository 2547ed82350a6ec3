// conflux_b200/csrc/tf32.cu -- the trailing update  C -= L * U  on the TF32 tensor cores (Hopper wgmma), the low-precision
// update of the mixed-precision drivers (cflx_lu_sv_mixed / cflx_chol_sv_mixed).  Never used by an FP64 factorisation.
//
//   * split: every row o of the K-major operand slabs (L^T / U of the LU, G / Bc of the Cholesky) gets ONE power-of-two
//     scale 2^e[o] with its largest magnitude in [0.5, 1) (frexp), so that FP64 inputs far outside FP32's exponent range
//     neither overflow nor flush.  s = x 2^-e (exact), hi = rna_tf32(fp32_rn(s)) and, for three terms, lo =
//     rna_tf32(fp32_rn(s - hi)), stored as FP32 bits [row][KP] with the K tail zero up to KP = K rounded up to 8.
//     rna_tf32 is cvt.rna.tf32.f32's rounding (to 10 explicit mantissa bits, ties away from zero), done on the bits so
//     that subnormal FP32 values round the same way (oracle/mixed_ref.py restates it bit for bit);
//   * product: TERMS = 1: acc += Ahi Bhi; TERMS = 3 (3xTF32): acc += Alo Bhi + Ahi Blo + Ahi Bhi, lo lo dropped; one
//     FP32 accumulator per element (wgmma.mma_async m64n128k8 .f32.tf32.tf32, both operands K-major);
//   * epilogue: C -= ldexp((double)acc, ea[m] + eb[n]) in place (alpha = -1, beta = 1 of the FP64 kernel).
//
// Kernel structure (persistent, one CTA per SM, 2 consumer warpgroups + 1 producer warp, CTA tile 128 x 128):
//   warp 8         TMA producer: 32-k chunks (one 128-byte swizzle row) of the A and B slabs (hi, and lo with three terms)
//                  fetched with cp.async.bulk.tensor.2d into a ring of stages; it runs ahead into the next tile while
//                  the consumers finish the current one;
//   warps 0-7      two warpgroups, 64 rows of the tile each, 64 FP32 accumulators per thread; a stage is released once
//                  the wgmma group that read it has completed (wait_group 1), so one group is always in flight.
#include <cuda.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>

#include "common.cuh"
#include "kernels.h"

namespace cflx {

namespace {
constexpr int TF_BM = 128, TF_BN = 128, TF_KC = 32;  // CTA tile; k-chunk of a stage (32 FP32 = one 128-byte row)
constexpr int TF_A_BYTES = TF_BM * TF_KC * 4, TF_B_BYTES = TF_BN * TF_KC * 4;
constexpr int TF_CONS_WARPS = 8;
constexpr int TF_THREADS = 32 * TF_CONS_WARPS + 32;
constexpr int TF_SPLIT_OUT = 32;  // outer indices per CTA of the split

template <int TERMS>
struct TfCfg {
    static constexpr int PARTS = TERMS == 1 ? 1 : 2;  // hi, or hi and lo, of both operands
    static constexpr int STAGE_BYTES = PARTS * (TF_A_BYTES + TF_B_BYTES);
    static constexpr int STAGES = TERMS == 1 ? 6 : 3;
    static constexpr size_t SMEM = 1024 /*alignment slack*/ + (size_t)STAGES * STAGE_BYTES + 128 /*barriers*/;
};

__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
            smem_u32(smem_dst)),
        "l"(map), "r"(c0), "r"(c1), "r"(smem_u32(bar))
        : "memory");
}
// shared-memory matrix descriptor of a K-major, 128-byte-swizzled operand tile (rows of 128 bytes, 8-row groups 1024 B
// apart): start address >> 4 | LBO (unused for swizzled K-major) = 1 at bit 16 | SBO = 1024 >> 4 at bit 32 |
// SWIZZLE_128B (1) at bit 62.  Stepping 8 TF32 (32 bytes) along K inside the swizzle atom adds 2 to the start field.
__device__ __forceinline__ uint64_t smem_desc_sw128(uint32_t saddr) {
    return (uint64_t)((saddr & 0x3FFFF) >> 4) | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// D(64 x 128, FP32 registers in the wgmma accumulator layout) += A(64 x 8, smem desc) * B(8 x 128, smem desc), TF32.
// Accumulator layout (thread T of the warpgroup, warp w = T / 32, lane l): d[4j + 2h + x] is row 16w + l/4 + 8h,
// column 8j + 2(l%4) + x.
__device__ __forceinline__ void wgmma_tf32_n128(float* d, uint64_t da, uint64_t db) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(1)
        : "memory");
}

struct TfArgs {
    int M, N, KC;      // C is M x N; KC = k chunks of TF_KC (the last one zero-filled beyond KP)
    int a_row0;        // first row of the A slab that belongs to row 0 of this C window
    int b_row0;        // first row of the B slab that belongs to column 0 of this C window
    double* C;         // in place: C -= A * B^T (both K-major)
    int64_t ldc;
    const int* ea;     // row exponents of A, indexed like the A rows
    const int* eb;     // row exponents of B, indexed like the B rows
    int tiles_m, tiles_n;
};

template <int TERMS>
__global__ void __launch_bounds__(TF_THREADS, 1)
tf32_gemm_kernel(const __grid_constant__ CUtensorMap mapAh, const __grid_constant__ CUtensorMap mapBh,
                 const __grid_constant__ CUtensorMap mapAl, const __grid_constant__ CUtensorMap mapBl, TfArgs g) {
    using Cfg = TfCfg<TERMS>;
    extern __shared__ unsigned char tf_smem_raw[];
    unsigned char* base = reinterpret_cast<unsigned char*>(((uintptr_t)tf_smem_raw + 1023) & ~(uintptr_t)1023);
    // stage st: A hi [128 rows][128 B], B hi [128][128 B], then (three terms) A lo, B lo
    uint64_t* full = reinterpret_cast<uint64_t*>(base + (size_t)Cfg::STAGES * Cfg::STAGE_BYTES);
    uint64_t* empty = full + Cfg::STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int ntiles = g.tiles_m * g.tiles_n;

    if (threadIdx.x == 0) {
        for (int i = 0; i < Cfg::STAGES; ++i) {
            mbar_init(&full[i], 1);
            mbar_init(&empty[i], TF_CONS_WARPS);
        }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == TF_CONS_WARPS) {
        // ================================================================== TMA producer
        if (lane == 0) {
            uint32_t q = 0;  // stage fills issued so far by this CTA
            for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
                const int m0 = (tile / g.tiles_n) * TF_BM, n0 = (tile % g.tiles_n) * TF_BN;
                for (int kc = 0; kc < g.KC; ++kc, ++q) {
                    const int st = q % Cfg::STAGES;
                    const uint32_t use = q / Cfg::STAGES;
                    if (use > 0) mbar_wait(&empty[st], (use - 1) & 1);
                    unsigned char* sa = base + (size_t)st * Cfg::STAGE_BYTES;
                    mbar_arrive_expect_tx(&full[st], (uint32_t)Cfg::STAGE_BYTES);
                    tma_load_2d(sa, &mapAh, kc * TF_KC, g.a_row0 + m0, &full[st]);
                    tma_load_2d(sa + TF_A_BYTES, &mapBh, kc * TF_KC, g.b_row0 + n0, &full[st]);
                    if constexpr (TERMS == 3) {
                        tma_load_2d(sa + TF_A_BYTES + TF_B_BYTES, &mapAl, kc * TF_KC, g.a_row0 + m0, &full[st]);
                        tma_load_2d(sa + 2 * TF_A_BYTES + TF_B_BYTES, &mapBl, kc * TF_KC, g.b_row0 + n0, &full[st]);
                    }
                }
            }
        }
        return;
    }

    // ====================================================================== consumers (two warpgroups)
    const int wg = warp >> 2;
    const uint32_t sbase = smem_u32(base);
    uint32_t q = 0;
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int m0 = (tile / g.tiles_n) * TF_BM, n0 = (tile % g.tiles_n) * TF_BN;
        const int r0 = m0 + 64 * wg + 16 * (warp & 3) + (lane >> 2);
        // the C rows this thread finishes, into L2 under the main loop: two lanes of each quad, a 32-byte sector each
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = r0 + 8 * h;
            if (row >= g.M) continue;
            const double* crow = g.C + (int64_t)row * g.ldc;
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const int col = n0 + 8 * j + 4 * (lane & 1);
                if ((lane & 3) < 2 && col < g.N) asm volatile("prefetch.global.L2 [%0];" ::"l"(crow + col));
            }
        }
        float acc[64];
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[i] = 0.f;
        int prev = -1;
        for (int kc = 0; kc < g.KC; ++kc, ++q) {
            const int st = q % Cfg::STAGES;
            mbar_wait(&full[st], (q / Cfg::STAGES) & 1);
            const uint32_t a_hi = sbase + st * Cfg::STAGE_BYTES + wg * (64 * 128);   // rows 64 wg .. of A
            const uint32_t b_hi = sbase + st * Cfg::STAGE_BYTES + TF_A_BYTES;
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < TF_KC / 8; ++k) {
                if constexpr (TERMS == 3) {
                    const uint32_t a_lo = a_hi + TF_A_BYTES + TF_B_BYTES, b_lo = b_hi + TF_A_BYTES + TF_B_BYTES;
                    wgmma_tf32_n128(acc, smem_desc_sw128(a_lo + 32 * k), smem_desc_sw128(b_hi + 32 * k));
                    wgmma_tf32_n128(acc, smem_desc_sw128(a_hi + 32 * k), smem_desc_sw128(b_lo + 32 * k));
                }
                wgmma_tf32_n128(acc, smem_desc_sw128(a_hi + 32 * k), smem_desc_sw128(b_hi + 32 * k));
            }
            wgmma_commit();
            wgmma_wait<1>();                                      // the group of the previous stage has completed
            if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
            prev = st;
        }
        wgmma_wait<0>();
        if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
        // ---- C -= ldexp(acc, ea + eb): each element has exactly one owner thread; C is read for a whole row first
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = r0 + 8 * h;
            if (row >= g.M) continue;
            const int er = g.ea[g.a_row0 + row];
            double* crow = g.C + (int64_t)row * g.ldc;
            double2 c[16];
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const int col = n0 + 8 * j + 2 * (lane & 3);
                if (col + 1 < g.N) c[j] = *reinterpret_cast<const double2*>(crow + col);
                else if (col < g.N) c[j].x = crow[col];
            }
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const int col = n0 + 8 * j + 2 * (lane & 3);
                if (col >= g.N) continue;
                c[j].x -= ldexp((double)acc[4 * j + 2 * h], er + g.eb[g.b_row0 + col]);
                if (col + 1 < g.N) {
                    c[j].y -= ldexp((double)acc[4 * j + 2 * h + 1], er + g.eb[g.b_row0 + col + 1]);
                    *reinterpret_cast<double2*>(crow + col) = c[j];
                } else {
                    crow[col] = c[j].x;
                }
            }
        }
    }
}

// cvt.rna.tf32.f32's rounding on the bits of a finite f: to 10 explicit mantissa bits, ties away from zero
__device__ __forceinline__ float rna_tf32(float f) {
    const uint32_t u = __float_as_uint(f);
    return __uint_as_float((u & 0x80000000u) | (((u & 0x7FFFFFFFu) + 0x1000u) & 0xFFFFE000u));
}

// src[k][o] (K x ld doubles, o = row of L / column of U) -> hi[o0 + o][k], lo[o0 + o][k] (FP32 bits, KP per row,
// zeros for K <= k < KP; lo only when lo != null), exps[o0 + o].  One CTA per 32 outer indices: pass 1 = largest
// magnitude per outer index, pass 2 = the split, transposed through shared memory.
__global__ void __launch_bounds__(256) tf32_split_kernel(const double* __restrict__ src, int64_t ld, int n_outer, int K,
                                                         int KP, float* __restrict__ hi, float* __restrict__ lo, int o0,
                                                         int* __restrict__ exps) {
    __shared__ float th[TF_SPLIT_OUT][TF_KC + 1], tl[TF_SPLIT_OUT][TF_KC + 1];
    __shared__ double red[8][TF_SPLIT_OUT];
    __shared__ int s_exp[TF_SPLIT_OUT];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int o = blockIdx.x * TF_SPLIT_OUT + tx;
    const bool valid = o < n_outer;
    double mx = 0.0;
    if (valid)
        for (int k = ty; k < K; k += 8) mx = fmax(mx, fabs(src[(int64_t)k * ld + o]));
    red[ty][tx] = mx;
    __syncthreads();
    if (ty == 0) {
#pragma unroll
        for (int i = 1; i < 8; ++i) mx = fmax(mx, red[i][tx]);
        int e = 0;
        if (mx > 0.0) frexp(mx, &e);  // mx = f 2^e, f in [0.5, 1): |x| 2^-e < 1 for the whole row
        s_exp[tx] = e;
        if (valid) exps[o0 + o] = e;
    }
    __syncthreads();
    const int e = s_exp[tx];
    for (int k0 = 0; k0 < KP; k0 += TF_KC) {
        for (int kk = ty; kk < TF_KC; kk += 8) {
            const int k = k0 + kk;
            const double s = (valid && k < K) ? ldexp(src[(int64_t)k * ld + o], -e) : 0.0;
            const float h = rna_tf32(__double2float_rn(s));
            th[tx][kk] = h;
            if (lo) tl[tx][kk] = rna_tf32(__double2float_rn(s - (double)h));
        }
        __syncthreads();
        for (int i = threadIdx.x; i < TF_SPLIT_OUT * TF_KC; i += 256) {
            const int r = i / TF_KC, c = i % TF_KC, k = k0 + c;
            const int oo = blockIdx.x * TF_SPLIT_OUT + r;
            if (oo < n_outer && k < KP) {
                hi[(int64_t)(o0 + oo) * KP + k] = th[r][c];
                if (lo) lo[(int64_t)(o0 + oo) * KP + k] = tl[r][c];
            }
        }
        __syncthreads();
    }
}

// ---------------------------------------------------------------------------------------------- host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess && p) fn = (EncodeTiledFn)p;
        cudaGetLastError();
    }
    return fn;
}
// slab: [rows][KP] FP32; box = 32 k x box_rows rows, 128-byte swizzle; what lies beyond KP or rows is read as zero
int make_slab_map(CUtensorMap* map, const float* slab, int KP, int rows, int box_rows) {
    EncodeTiledFn fn = encode_fn();
    if (!fn) {
        set_last_error("cuTensorMapEncodeTiled is not available from the driver");
        return CFLX_ERR_CUDA;
    }
    cuuint64_t dims[2] = {(cuuint64_t)KP, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)KP * sizeof(float)};
    cuuint32_t box[2] = {(cuuint32_t)TF_KC, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void*)slab, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_last_error("cuTensorMapEncodeTiled failed (%d) for KP=%d rows=%d", (int)r, KP, rows);
        return CFLX_ERR_CUDA;
    }
    return CFLX_OK;
}

template <int TERMS>
int tf32_kernel_setup() {
    static PerDeviceMax cfg;
    CFLX_CUDA(cfg.raise(TfCfg<TERMS>::SMEM, [&] {
        return cudaFuncSetAttribute(tf32_gemm_kernel<TERMS>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    (int)TfCfg<TERMS>::SMEM);
    }));
    return CFLX_OK;
}
}  // namespace

struct Tf32Workspace::Maps {
    CUtensorMap ah, bh, al, bl;
};

Tf32Workspace::Tf32Workspace() = default;
Tf32Workspace::~Tf32Workspace() = default;

int tf32_workspace_create(Tf32Workspace* ws, int max_rows, int max_cols, int K) {
    if (K <= 0) {
        set_last_error("tf32: contraction length %d unsupported", K);
        return CFLX_ERR_UNSUPPORTED;
    }
    ws->K = K;
    ws->KP = (int)round_up(K, 8);
    ws->cap_a = (int)round_up(std::max(max_rows, 1), TF_BM);
    ws->cap_b = (int)round_up(std::max(max_cols, 1), TF_BN);
    const size_t na = (size_t)ws->cap_a * ws->KP, nb = (size_t)ws->cap_b * ws->KP;
    for (auto* b : {&ws->hiA, &ws->loA}) {
        CFLX_TRY(b->alloc_exact(na));
        CFLX_CUDA(cudaMemset(b->p, 0, na * sizeof(float)));
    }
    for (auto* b : {&ws->hiB, &ws->loB}) {
        CFLX_TRY(b->alloc_exact(nb));
        CFLX_CUDA(cudaMemset(b->p, 0, nb * sizeof(float)));
    }
    CFLX_TRY(ws->ea.alloc_exact(ws->cap_a));
    CFLX_TRY(ws->eb.alloc_exact(ws->cap_b));
    CFLX_CUDA(cudaMemset(ws->ea, 0, sizeof(int) * ws->cap_a));
    CFLX_CUDA(cudaMemset(ws->eb, 0, sizeof(int) * ws->cap_b));
    ws->maps = std::make_unique<Tf32Workspace::Maps>();
    CFLX_TRY(make_slab_map(&ws->maps->ah, ws->hiA, ws->KP, ws->cap_a, TF_BM));
    CFLX_TRY(make_slab_map(&ws->maps->al, ws->loA, ws->KP, ws->cap_a, TF_BM));
    CFLX_TRY(make_slab_map(&ws->maps->bh, ws->hiB, ws->KP, ws->cap_b, TF_BN));
    CFLX_TRY(make_slab_map(&ws->maps->bl, ws->loB, ws->KP, ws->cap_b, TF_BN));
    CFLX_TRY(tf32_kernel_setup<1>());
    CFLX_TRY(tf32_kernel_setup<3>());
    int dev = 0;
    CFLX_CUDA(cudaGetDevice(&dev));
    CFLX_CUDA(cudaDeviceGetAttribute(&ws->sms, cudaDevAttrMultiProcessorCount, dev));
    return CFLX_OK;
}

// rows [0, n) of L^T (LT[k][row], ld) -> the A slabs
int tf32_split_a(Tf32Workspace* ws, int terms, const double* LT, int64_t ld, int n, cudaStream_t s) {
    if (n <= 0) return CFLX_OK;
    if (n > ws->cap_a || (terms != 1 && terms != 3)) return CFLX_ERR_ARG;
    tf32_split_kernel<<<(n + TF_SPLIT_OUT - 1) / TF_SPLIT_OUT, 256, 0, s>>>(LT, ld, n, ws->K, ws->KP, ws->hiA,
                                                                           terms == 3 ? ws->loA.p : nullptr, 0, ws->ea);
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}
// columns [col0, col0 + n) of U (U[k][col], ld) -> the B slabs, rows col0..
int tf32_split_b(Tf32Workspace* ws, int terms, const double* U, int64_t ld, int col0, int n, cudaStream_t s) {
    if (n <= 0) return CFLX_OK;
    if (col0 < 0 || col0 + n > ws->cap_b || (terms != 1 && terms != 3)) return CFLX_ERR_ARG;
    tf32_split_kernel<<<(n + TF_SPLIT_OUT - 1) / TF_SPLIT_OUT, 256, 0, s>>>(U + col0, ld, n, ws->K, ws->KP, ws->hiB,
                                                                           terms == 3 ? ws->loB.p : nullptr, col0, ws->eb);
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}
// C[0..M) x [0..N) -= (rows row0..row0+M of the A slabs) * (rows col0..col0+N of the B slabs)^T
int launch_tf32_gemm(Tf32Workspace* ws, int terms, int M, int N, int row0, int col0, double* C, int64_t ldc, int max_ctas,
                     cudaStream_t s) {
    if (M <= 0 || N <= 0) return CFLX_OK;
    if ((terms != 1 && terms != 3) || (ldc & 1) || ((uintptr_t)C & 15) || col0 < 0 || row0 < 0 ||
        row0 + M > ws->cap_a || col0 + N > ws->cap_b) {
        set_last_error("tf32_gemm: unsupported window terms=%d M=%d N=%d row0=%d col0=%d ldc=%lld", terms, M, N, row0, col0,
                       (long long)ldc);
        return CFLX_ERR_UNSUPPORTED;
    }
    TfArgs g{};
    g.M = M; g.N = N;
    g.KC = (ws->KP + TF_KC - 1) / TF_KC;
    g.a_row0 = row0;
    g.b_row0 = col0;
    g.C = C; g.ldc = ldc;
    g.ea = ws->ea; g.eb = ws->eb;
    g.tiles_m = (M + TF_BM - 1) / TF_BM;
    g.tiles_n = (N + TF_BN - 1) / TF_BN;
    int grid = g.tiles_m * g.tiles_n;
    int cap = ws->sms;
    if (max_ctas > 0 && max_ctas < cap) cap = max_ctas;
    if (grid > cap) grid = cap;
    const Tf32Workspace::Maps& m = *ws->maps;
    if (terms == 1) tf32_gemm_kernel<1><<<grid, TF_THREADS, TfCfg<1>::SMEM, s>>>(m.ah, m.bh, m.al, m.bl, g);
    else tf32_gemm_kernel<3><<<grid, TF_THREADS, TfCfg<3>::SMEM, s>>>(m.ah, m.bh, m.al, m.bl, g);
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}

}  // namespace cflx
