// conflux_b200/csrc/ozaki.cu -- the trailing update  C -= L * U  as exact int8 tensor-core products (Hopper wgmma).
//
// Replaces cblas_dgemm at conflux_opt.hpp:1628-1632 of the reference on the path selected by CFLX_GEMM=ozaki (gemm.cu's
// FP64 DMMA kernel is the default trailing update on H100 and serves the TRSM sweeps).  wgmma has no f64 kind, so FP64
// accuracy is recovered with error-free slicing (Ozaki scheme):
//   * every row m of L and every column n of U gets ONE power-of-two scale 2^ea[m] / 2^eb[n] (its largest magnitude);
//   * the scaled entries are cut into S = 8 signed digits (first 6 bits, then 7 bits each, round-to-nearest so every
//     digit fits [-64, 64]): x = 2^(e-6) * sum_s d_s 2^(-7s), exact to 55 bits relative to the row/column maximum;
//   * every digit-plane product  sum_k da_s[m][k] * db_t[k][n]  is an EXACT int8 x int8 -> int32 GEMM
//     (wgmma.mma_async .s32.s8.s8, accumulators in registers); the planes with s + t = g share one accumulator (their
//     weight 2^(-7g) is the same; at most 8 products of <= 2^12 * K, K <= 512: < 2^25), only g <= 7 is kept (36 MMAs);
//   * the epilogue recombines  sum_g 2^(-7g) acc_g  in FP64 in the order g = 0, 1, ..., 7, applies 2^(ea+eb-12) and
//     subtracts from C in place.
// The neglected planes (g >= 8) are below 2^-56 of |row max| * |column max| per term: the same order as the rounding of
// a native FP64 dot product of that length (tools/ozaki_study.py: residual and pivots unchanged at 8 slices).
//
// Kernel structure (one CTA per SM, 2 consumer warpgroups + 1 producer warp, CTA tile 128 x 64):
//   warp 8         TMA producer: digit planes are K-major int8 ([plane][row][K], 64-byte swizzled boxes of 64 k) fetched
//                  with cp.async.bulk.tensor.3d through two tensor maps into a two-stage ring; one stage holds one 64-k
//                  chunk of every plane the current pass needs, for both operands;
//   warps 0-7      two warpgroups, 64 rows of the tile each.  The 8 groups are accumulated in passes of OZ_GP groups
//                  (int32 registers: OZ_GP x 32 per thread); after each pass the finished groups are folded into the
//                  FP64 running sum in group order, so the recombination is the same sequence of roundings as a single
//                  pass.  The B planes t, t+1, ... of a stage are contiguous 64-row tiles and the accumulators of their
//                  groups are contiguous registers: all planes of one A_s in the pass go through ONE wgmma of
//                  N = 64 * planes, so A_s is read from shared memory once per pass and k step.
#include <algorithm>

#include "kernels.h"
#include "wgmma.cuh"

namespace cflx {

namespace {
constexpr int OZ_S = 8;                               // digit planes per operand
constexpr int OZ_BM = 128, OZ_BN = 64, OZ_KC = 64;    // CTA tile, k-chunk of a pipeline stage (bytes = int8 elements)
constexpr int OZ_GP = 3;                              // accumulator groups per pass
constexpr int OZ_NPASS = (OZ_S + OZ_GP - 1) / OZ_GP;
constexpr int OZ_STAGES = 2;
constexpr int OZ_A_BYTES = OZ_BM * OZ_KC, OZ_B_BYTES = OZ_BN * OZ_KC;   // one plane of one stage
constexpr int OZ_STAGE_BYTES = OZ_S * (OZ_A_BYTES + OZ_B_BYTES);
constexpr int OZ_CONS_WARPS = 8;
constexpr int OZ_THREADS = 32 * OZ_CONS_WARPS + 32;
constexpr size_t OZ_SMEM = 1024 /*alignment slack*/ + (size_t)OZ_STAGES * OZ_STAGE_BYTES + 64 /*barriers*/;
constexpr int OZ_SPLIT_KC = 128;                      // k-chunk of the digit-plane split (K is a multiple of it)

// D(64 x n, int32 registers in the wgmma accumulator layout) += A(64 x 32, smem desc) * B(32 x n, smem desc), int8.
// Accumulator layout (thread T of the warpgroup, warp w = T / 32, lane l): d[4j + 2h + x] is row 16w + l/4 + 8h,
// column 8j + 2(l%4) + x.
__device__ __forceinline__ void wgmma_s8_n64(int* d, uint64_t da, uint64_t db) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k32.s32.s8.s8 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p;\n\t}"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31])
        : "l"(da), "l"(db), "r"(1)
        : "memory");
}
__device__ __forceinline__ void wgmma_s8_n128(int* d, uint64_t da, uint64_t db) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k32.s32.s8.s8 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p;\n\t}"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
        : "l"(da), "l"(db), "r"(1)
        : "memory");
}
__device__ __forceinline__ void wgmma_s8_n192(int* d, uint64_t da, uint64_t db) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %98, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n192k32.s32.s8.s8 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95}, %96, %97, p;\n\t}"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63]), "+r"(d[64]), "+r"(d[65]), "+r"(d[66]), "+r"(d[67]), "+r"(d[68]), "+r"(d[69]), "+r"(d[70]), "+r"(d[71]), "+r"(d[72]), "+r"(d[73]), "+r"(d[74]), "+r"(d[75]), "+r"(d[76]), "+r"(d[77]), "+r"(d[78]), "+r"(d[79]), "+r"(d[80]), "+r"(d[81]), "+r"(d[82]), "+r"(d[83]), "+r"(d[84]), "+r"(d[85]), "+r"(d[86]), "+r"(d[87]), "+r"(d[88]), "+r"(d[89]), "+r"(d[90]), "+r"(d[91]), "+r"(d[92]), "+r"(d[93]), "+r"(d[94]), "+r"(d[95])
        : "l"(da), "l"(db), "r"(1)
        : "memory");
}
__device__ __forceinline__ void wgmma_s8_n256(int* d, uint64_t da, uint64_t db) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k32.s32.s8.s8 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p;\n\t}"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63]), "+r"(d[64]), "+r"(d[65]), "+r"(d[66]), "+r"(d[67]), "+r"(d[68]), "+r"(d[69]), "+r"(d[70]), "+r"(d[71]), "+r"(d[72]), "+r"(d[73]), "+r"(d[74]), "+r"(d[75]), "+r"(d[76]), "+r"(d[77]), "+r"(d[78]), "+r"(d[79]), "+r"(d[80]), "+r"(d[81]), "+r"(d[82]), "+r"(d[83]), "+r"(d[84]), "+r"(d[85]), "+r"(d[86]), "+r"(d[87]), "+r"(d[88]), "+r"(d[89]), "+r"(d[90]), "+r"(d[91]), "+r"(d[92]), "+r"(d[93]), "+r"(d[94]), "+r"(d[95]), "+r"(d[96]), "+r"(d[97]), "+r"(d[98]), "+r"(d[99]), "+r"(d[100]), "+r"(d[101]), "+r"(d[102]), "+r"(d[103]), "+r"(d[104]), "+r"(d[105]), "+r"(d[106]), "+r"(d[107]), "+r"(d[108]), "+r"(d[109]), "+r"(d[110]), "+r"(d[111]), "+r"(d[112]), "+r"(d[113]), "+r"(d[114]), "+r"(d[115]), "+r"(d[116]), "+r"(d[117]), "+r"(d[118]), "+r"(d[119]), "+r"(d[120]), "+r"(d[121]), "+r"(d[122]), "+r"(d[123]), "+r"(d[124]), "+r"(d[125]), "+r"(d[126]), "+r"(d[127])
        : "l"(da), "l"(db), "r"(1)
        : "memory");
}

// acc[0 .. 32 * planes) += A * (planes consecutive B tiles of 64 rows)
template <int PLANES>
__device__ __forceinline__ void wgmma_s8(int* acc, uint64_t da, uint64_t db) {
    if constexpr (PLANES == 1) wgmma_s8_n64(acc, da, db);
    else if constexpr (PLANES == 2) wgmma_s8_n128(acc, da, db);
    else if constexpr (PLANES == 3) wgmma_s8_n192(acc, da, db);
    else wgmma_s8_n256(acc, da, db);
}

__host__ __device__ constexpr double pow2c(int e) {  // compile-time 2^e, e <= 0
    double x = 1.0;
    for (int i = 0; i < -e; ++i) x *= 0.5;
    return x;
}
__device__ __forceinline__ double pow2i(int e) { return __longlong_as_double((long long)(1023 + e) << 52); }  // |e| < 1022

struct OzArgs {
    int M, N, K;           // C is M x N, K = contraction length (multiple of 128)
    int a_row0;            // first row of the A planes that belongs to row 0 of this C window
    int b_row0;            // first row of the B planes that belongs to column 0 of this C window
    double* C;             // in place: C -= A^T-planes * B-planes
    int64_t ldc;
    const int* ea;         // [M]   row exponents of A
    const int* eb;         // [...] column exponents of B, indexed like the B planes (b_row0 + n)
    int tiles_m, tiles_n;
};

// the plane products of groups [G0, G0 + OZ_GP) for one 64-k chunk held in one stage: for every A plane s, the B planes
// t = max(0, G0 - s) .. G1 - s in one instruction (their groups s + t are consecutive accumulators)
template <int G0, int S>
__device__ __forceinline__ void pass_products(int* acc, uint32_t a_base, uint32_t b_base) {
    constexpr int G1 = (G0 + OZ_GP < OZ_S ? G0 + OZ_GP : OZ_S) - 1;
    if constexpr (S <= G1) {
        constexpr int T_LO = G0 - S > 0 ? G0 - S : 0;
        constexpr int PLANES = G1 - S - T_LO + 1;
#pragma unroll
        for (int k = 0; k < OZ_KC / 32; ++k)
            wgmma_s8<PLANES>(acc + 32 * (S + T_LO - G0), smem_desc<64>(a_base + S * OZ_A_BYTES + 32 * k),
                             smem_desc<64>(b_base + T_LO * OZ_B_BYTES + 32 * k));
        pass_products<G0, S + 1>(acc, a_base, b_base);
    }
}

template <int P>
__device__ __forceinline__ void consume_pass(const OzArgs& g, uint64_t* full, uint64_t* empty, uint32_t sbase, int wg, int lane,
                                             uint32_t& q, double (&sum)[32]) {
    if constexpr (P < OZ_NPASS) {
        constexpr int G0 = P * OZ_GP;
        constexpr int NG = (G0 + OZ_GP < OZ_S ? OZ_GP : OZ_S - G0);
        int acc[OZ_GP * 32];
#pragma unroll
        for (int i = 0; i < OZ_GP * 32; ++i) acc[i] = 0;
        const int KC = g.K / OZ_KC;
        for (int kc = 0; kc < KC; ++kc, ++q) {
            const int st = q % OZ_STAGES;
            mbar_wait(&full[st], (q / OZ_STAGES) & 1);
            const uint32_t a_base = sbase + st * OZ_STAGE_BYTES + wg * (64 * OZ_KC);   // rows 64 wg .. of every A plane
            const uint32_t b_base = sbase + st * OZ_STAGE_BYTES + OZ_S * OZ_A_BYTES;
            wgmma_fence();
            pass_products<G0, 0>(acc, a_base, b_base);
            wgmma_commit();
            wgmma_wait<0>();
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[st]);                  // this warp is done with the stage
        }
#pragma unroll
        for (int gi = 0; gi < NG; ++gi) {
            const double w = pow2c(-7 * (G0 + gi));
#pragma unroll
            for (int i = 0; i < 32; ++i) {
                // exact int32 -> double without the conversion pipe: 2^52 + 2^31 + x, then subtract the bias
                const double x = __hiloint2double(0x43300000, acc[32 * gi + i] ^ 0x80000000) - 4503601774854144.0;
                sum[i] = fma(x, w, sum[i]);
            }
        }
        consume_pass<P + 1>(g, full, empty, sbase, wg, lane, q, sum);
    }
}

__global__ void __launch_bounds__(OZ_THREADS, 1)
ozaki_gemm_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB, OzArgs g) {
    extern __shared__ unsigned char oz_smem_raw[];
    unsigned char* base = reinterpret_cast<unsigned char*>(((uintptr_t)oz_smem_raw + 1023) & ~(uintptr_t)1023);
    // stage st: A planes [8][128 rows][64 B], then B planes [8][64 rows][64 B]
    uint64_t* full = reinterpret_cast<uint64_t*>(base + (size_t)OZ_STAGES * OZ_STAGE_BYTES);
    uint64_t* empty = full + OZ_STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int ntiles = g.tiles_m * g.tiles_n;
    const int KC = g.K / OZ_KC;

    if (threadIdx.x == 0) {
        for (int i = 0; i < OZ_STAGES; ++i) {
            mbar_init(&full[i], 1);
            mbar_init(&empty[i], OZ_CONS_WARPS);
        }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == OZ_CONS_WARPS) {
        // ================================================================== TMA producer
        if (lane == 0) {
            uint32_t q = 0;  // stage fills issued so far by this CTA
            for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
                const int m0 = (tile / g.tiles_n) * OZ_BM, n0 = (tile % g.tiles_n) * OZ_BN;
                for (int p = 0; p < OZ_NPASS; ++p) {
                    const int np = (p + 1) * OZ_GP < OZ_S ? (p + 1) * OZ_GP : OZ_S;   // the pass needs planes 0 .. np-1 of both operands
                    for (int kc = 0; kc < KC; ++kc, ++q) {
                        const int st = q % OZ_STAGES;
                        const uint32_t use = q / OZ_STAGES;
                        if (use > 0) mbar_wait(&empty[st], (use - 1) & 1);
                        unsigned char* sa = base + (size_t)st * OZ_STAGE_BYTES;
                        unsigned char* sb = sa + OZ_S * OZ_A_BYTES;
                        mbar_arrive_expect_tx(&full[st], (uint32_t)(np * (OZ_A_BYTES + OZ_B_BYTES)));
                        for (int t = 0; t < np; ++t) {
                            tma_load_3d(sa + t * OZ_A_BYTES, &mapA, kc * OZ_KC, g.a_row0 + m0, t, &full[st]);
                            tma_load_3d(sb + t * OZ_B_BYTES, &mapB, kc * OZ_KC, g.b_row0 + n0, t, &full[st]);
                        }
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
        const int m0 = (tile / g.tiles_n) * OZ_BM, n0 = (tile % g.tiles_n) * OZ_BN;
        double sum[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) sum[i] = 0.0;
        consume_pass<0>(g, full, empty, sbase, wg, lane, q, sum);
        // ---- C -= sum * 2^(ea - 12) * 2^eb, as C + (sum * -2^(ea - 12)) * 2^eb: each element has exactly one owner thread
        const int r0 = m0 + 64 * wg + 16 * (warp & 3) + (lane >> 2);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = r0 + 8 * h;
            if (row >= g.M) continue;
            const double sr = -pow2i(g.ea[g.a_row0 + row] - 12);
            double* crow = g.C + (int64_t)row * g.ldc;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int col = n0 + 8 * j + 2 * (lane & 3);
                if (col >= g.N) continue;                              // N is even: col + 1 < N too
                double2 c = *reinterpret_cast<const double2*>(crow + col);
                c.x += (sum[4 * j + 2 * h] * sr) * pow2i(g.eb[g.b_row0 + col]);
                c.y += (sum[4 * j + 2 * h + 1] * sr) * pow2i(g.eb[g.b_row0 + col + 1]);
                *reinterpret_cast<double2*>(crow + col) = c;
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------- raw wgmma rate probe
// Back-to-back wgmma m64 x n x 32 (int8) on resident shared-memory tiles, two warpgroups per CTA, one CTA per SM (no TMA,
// no epilogue): the tensor cores' own int8 rate, the ceiling of the digit-plane GEMM.
template <int PLANES>
__global__ void __launch_bounds__(256, 1) wgmma_peak_kernel(int iters, int* sink) {
    extern __shared__ unsigned char pk_smem_raw[];
    unsigned char* base = reinterpret_cast<unsigned char*>(((uintptr_t)pk_smem_raw + 1023) & ~(uintptr_t)1023);
    for (int i = threadIdx.x; i < (4096 + 16384) / 4; i += blockDim.x) reinterpret_cast<uint32_t*>(base)[i] = 0x01010101u * (i & 3);
    fence_proxy_async();
    __syncthreads();
    int acc[32 * PLANES];
#pragma unroll
    for (int i = 0; i < 32 * PLANES; ++i) acc[i] = 0;
    const uint32_t a = smem_u32(base), b = smem_u32(base + 4096);
    wgmma_fence();
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int k = 0; k < 2; ++k) wgmma_s8<PLANES>(acc, smem_desc<64>(a + 32 * k), smem_desc<64>(b + 32 * k));
        wgmma_commit();
        wgmma_wait<1>();
    }
    wgmma_wait<0>();
    int x = 0;
#pragma unroll
    for (int i = 0; i < 32 * PLANES; ++i) x ^= acc[i];
    if (x == 0x7fffffff) *sink = x;   // keeps the MMAs alive
}

// ---------------------------------------------------------------------------------------------- digit planes
// src[k][o] (K x ld doubles, o = row of L / column of U) -> planes[s][o0 + o][k] int8 (K contiguous), exps[o0 + o].
// One CTA per 32 outer indices: pass 1 = largest magnitude per outer index, pass 2 = digits, transposed through smem.
constexpr int OZ_SPLIT_OUT = 32;
__global__ void __launch_bounds__(256) ozaki_split_kernel(const double* __restrict__ src, int64_t ld, int n_outer, int K,
                                                          int8_t* __restrict__ planes, int64_t plane_stride, int o0,
                                                          int* __restrict__ exps) {
    constexpr int PITCH = OZ_SPLIT_KC + 4;  // bytes per smem row: 33 words, conflict-free byte scatter
    __shared__ __align__(16) unsigned char tile[OZ_S][OZ_SPLIT_OUT][PITCH];
    __shared__ double red[8][OZ_SPLIT_OUT];
    __shared__ int s_exp[OZ_SPLIT_OUT];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int o = blockIdx.x * OZ_SPLIT_OUT + tx;
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
        if (mx > 0.0) frexp(mx, &e);  // mx = f * 2^e, f in [0.5, 1): |x| * 2^-e < 1 for the whole row
        s_exp[tx] = e;
        if (valid) exps[o0 + o] = e;
    }
    __syncthreads();
    const double inv = pow2i(-s_exp[tx]);
    for (int k0 = 0; k0 < K; k0 += OZ_SPLIT_KC) {
        for (int kk = ty; kk < OZ_SPLIT_KC; kk += 8) {
            double r = valid ? src[(int64_t)(k0 + kk) * ld + o] * inv : 0.0;
            r *= 64.0;  // first digit: 6 bits
#pragma unroll
            for (int s = 0; s < OZ_S; ++s) {
                const double d = rint(r);
                tile[s][tx][kk] = (unsigned char)(signed char)(int)d;
                r = (r - d) * 128.0;
            }
        }
        __syncthreads();
        // write-out: plane s, outer row, 128 contiguous bytes = 8 x 16 B
        for (int e = threadIdx.x; e < OZ_S * OZ_SPLIT_OUT * 8; e += 256) {
            const int s = e / (OZ_SPLIT_OUT * 8), rowi = (e / 8) % OZ_SPLIT_OUT, c16 = e % 8;
            const int oo = blockIdx.x * OZ_SPLIT_OUT + rowi;
            if (oo < n_outer) {
                const uint32_t* w = reinterpret_cast<const uint32_t*>(&tile[s][rowi][c16 * 16]);
                uint4 v = make_uint4(w[0], w[1], w[2], w[3]);
                *reinterpret_cast<uint4*>(planes + (int64_t)s * plane_stride + (int64_t)(o0 + oo) * K + k0 + c16 * 16) = v;
            }
        }
        __syncthreads();
    }
}

// ---------------------------------------------------------------------------------------------- host side
// planes: [OZ_S][cap_rows][K] int8; box = 64 bytes of k x box_rows rows of one plane, 64-byte swizzle
int make_plane_map(CUtensorMap* map, const int8_t* planes, int K, int cap_rows, int box_rows) {
    const cuuint64_t dims[3] = {(cuuint64_t)K, (cuuint64_t)cap_rows, (cuuint64_t)OZ_S};
    const cuuint64_t strides[2] = {(cuuint64_t)K, (cuuint64_t)K * (cuuint64_t)cap_rows};
    const cuuint32_t box[3] = {(cuuint32_t)OZ_KC, (cuuint32_t)box_rows, 1};
    return make_tensor_map(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, planes, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_64B);
}
}  // namespace

struct OzakiWorkspace::Maps {
    CUtensorMap a, b;
};

OzakiWorkspace::OzakiWorkspace() = default;
OzakiWorkspace::~OzakiWorkspace() = default;

int ozaki_workspace_create(OzakiWorkspace* ws, int max_rows, int max_cols, int K) {
    if (K <= 0 || K % OZ_SPLIT_KC != 0 || K > 512) {
        set_last_error("ozaki: contraction length %d unsupported (multiple of 128, <= 512)", K);
        return CFLX_ERR_UNSUPPORTED;
    }
    CFLX_TRY(ws->init(max_rows, max_cols, K, OZ_BM, OZ_BN));
    CFLX_TRY(ws->planesA.alloc_exact((size_t)OZ_S * ws->cap_a * K));
    CFLX_TRY(ws->planesB.alloc_exact((size_t)OZ_S * ws->cap_b * K));
    CFLX_CUDA(cudaMemset(ws->planesA, 0, (size_t)OZ_S * ws->cap_a * K));
    CFLX_CUDA(cudaMemset(ws->planesB, 0, (size_t)OZ_S * ws->cap_b * K));
    ws->maps = std::make_unique<OzakiWorkspace::Maps>();
    CFLX_TRY(make_plane_map(&ws->maps->a, ws->planesA, K, ws->cap_a, OZ_BM));
    CFLX_TRY(make_plane_map(&ws->maps->b, ws->planesB, K, ws->cap_b, OZ_BN));
    static PerDeviceMax cfg;
    CFLX_CUDA(cfg.raise(OZ_SMEM, [&] {
        return cudaFuncSetAttribute(ozaki_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)OZ_SMEM);
    }));
    return CFLX_OK;
}

// Tera-MACs/s of back-to-back int8 wgmma 64 x n x 32 instructions (n = 64, 128, 192 or 256), two warpgroups per CTA,
// one CTA per SM.
int wgmma_peak_probe(int n, double* tmacs_out) {
    void (*kern)(int, int*) = n == 64 ? wgmma_peak_kernel<1> : n == 128 ? wgmma_peak_kernel<2> : n == 192 ? wgmma_peak_kernel<3>
                            : n == 256 ? wgmma_peak_kernel<4> : nullptr;
    if (!kern) return CFLX_ERR_ARG;
    int dev = 0, sms = 0;
    CFLX_CUDA(cudaGetDevice(&dev));
    CFLX_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const size_t smem = 1024 + 4096 + 16384;
    CFLX_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    DevBuf<> sink;
    CFLX_TRY(sink.alloc(sizeof(int)));
    Events<2> ev;
    CFLX_TRY(ev.create());
    const int iters = 20000;
    double best = 0;
    for (int rep = 0; rep < 3; ++rep) {
        CFLX_CUDA(cudaEventRecord(ev[0]));
        kern<<<sms, 256, smem>>>(iters, sink.as<int>());
        CFLX_CUDA(cudaEventRecord(ev[1]));
        CFLX_CUDA(cudaEventSynchronize(ev[1]));
        float ms = 0;
        CFLX_CUDA(cudaEventElapsedTime(&ms, ev[0], ev[1]));
        const double macs = (double)sms * 2 * iters * 2 * 64.0 * n * 32.0;
        best = std::max(best, macs / (ms * 1e-3) / 1e12);
    }
    CFLX_CUDA(cudaGetLastError());
    *tmacs_out = best;
    return CFLX_OK;
}

// digit planes of rows [0, n) of L^T (LT[k][row], ld) -> A planes
int ozaki_split_a(OzakiWorkspace* ws, const double* LT, int64_t ld, int n, cudaStream_t s) {
    if (n <= 0) return CFLX_OK;
    if (n > ws->cap_a) return CFLX_ERR_ARG;
    ozaki_split_kernel<<<(n + OZ_SPLIT_OUT - 1) / OZ_SPLIT_OUT, 256, 0, s>>>(LT, ld, n, ws->K, ws->planesA, (int64_t)ws->cap_a * ws->K, 0, ws->ea);
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}
// digit planes of columns [col0, col0 + n) of U (U[k][col], ld) -> B planes, rows col0..
int ozaki_split_b(OzakiWorkspace* ws, const double* U, int64_t ld, int col0, int n, cudaStream_t s) {
    if (n <= 0) return CFLX_OK;
    if (col0 < 0 || col0 + n > ws->cap_b) return CFLX_ERR_ARG;
    ozaki_split_kernel<<<(n + OZ_SPLIT_OUT - 1) / OZ_SPLIT_OUT, 256, 0, s>>>(U + col0, ld, n, ws->K, ws->planesB, (int64_t)ws->cap_b * ws->K, col0, ws->eb);
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}
// C[0..M) x [0..N) -= (rows row0..row0+M of the A planes) * (rows col0..col0+N of the B planes)
int launch_ozaki_gemm(OzakiWorkspace* ws, int M, int N, int row0, int col0, double* C, int64_t ldc, int max_ctas, cudaStream_t s) {
    if (M <= 0 || N <= 0) return CFLX_OK;
    if ((N & 1) || (ldc & 1) || col0 < 0 || row0 < 0 || row0 + M > ws->cap_a || col0 + N > ws->cap_b) {
        set_last_error("ozaki_gemm: unsupported window M=%d N=%d row0=%d col0=%d ldc=%lld", M, N, row0, col0, (long long)ldc);
        return CFLX_ERR_UNSUPPORTED;
    }
    OzArgs g{};
    g.M = M; g.N = N; g.K = ws->K;
    g.a_row0 = row0;
    g.b_row0 = col0;
    g.C = C; g.ldc = ldc;
    g.ea = ws->ea; g.eb = ws->eb;
    g.tiles_m = (M + OZ_BM - 1) / OZ_BM;
    g.tiles_n = (N + OZ_BN - 1) / OZ_BN;
    ozaki_gemm_kernel<<<ws->grid(g.tiles_m * g.tiles_n, max_ctas), OZ_THREADS, OZ_SMEM, s>>>(ws->maps->a, ws->maps->b, g);
    CFLX_CUDA(cudaGetLastError());
    return CFLX_OK;
}

}  // namespace cflx
