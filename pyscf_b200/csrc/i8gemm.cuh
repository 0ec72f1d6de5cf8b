// i8gemm.cuh — FP64-accurate GEMM on the Hopper tensor cores (wgmma, s8 x s8 -> s32) by error-free slicing (Ozaki
// scheme): the DF-K contractions of pyscf/df/df_jk.py:373-380 (AO2MOnr_e2_drv's dsymm and lib.dot/NPdgemm) executed as exact
// int8 x int8 -> int32 slice products.
//
//   C[m,n] (+)= sum_k A[m,k] B[n,k]            A: [M,K], B: [N,K] fp64, both K-major (row-major, K contiguous)
//
// 1. the slicing kernels below scale every row by 2^-E (E = ceil(log2 max|row|)) and cut it into NS signed 7-bit slices
//        a = 2^E ( q0 2^-6 + q1 2^-13 + ... + q_{NS-1} 2^-(6+7(NS-1)) ) + tail,  |q| <= 64.
// 2. i8gemm_kernel: for every slice-pair group g = k+l (same power of two) the products A_k B_l^T are accumulated EXACTLY
//    in int32 registers by wgmma.mma_async (operands TMA-loaded into 128B-swizzled shared memory through mbarrier rings);
//    all groups of a tile stay resident, each A_k tile is multiplied once with its stacked B slices.  The groups are then
//    converted to fp64, weighted by 2^(-12-7g) and summed, smallest weight first; the epilogue applies the row / column
//    exponents 2^(Ea[m]+Eb[n]) once per output element.
// Only pairs with k+l < NS are formed (the rest is below the slice truncation): NS(NS+1)/2 slice GEMMs.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200jk {
namespace i8g {

constexpr int BM = 128;        // rows of an output tile: two consumer warpgroups of 64 rows (wgmma M = 64)
constexpr int BN = 32;         // columns of an output tile = rows of one B slice tile
constexpr int BK = 128;        // bytes (= int8 elements) of K per pipeline stage: one 128B swizzle row
constexpr int UK = 32;         // K per wgmma (s8)
constexpr int MAXS = 8;        // max slices
constexpr int NSA = 8;         // depth of the A ring (one A_k slice tile per stage)
constexpr int NSB = 2;         // depth of the B ring (all ns slices of one K block per stage)
constexpr int A_STAGE_BYTES = BM * BK;
constexpr int B_SLICE_BYTES = BN * BK;
constexpr int BAR_BYTES = 256;
__host__ __device__ constexpr int smem_bytes(int ns) { return NSA * A_STAGE_BYTES + NSB * ns * B_SLICE_BYTES + BAR_BYTES + 1024 /*align*/; }
constexpr int NTHREADS = 384;  // warpgroup 0: TMA producer (one thread), warpgroups 1, 2: wgmma + epilogue (64 rows each)
constexpr int NCONSUMER_WARPS = 8;

struct GemmParams {
    int M, N, Kp;          // Kp: padded K (multiple of BK)
    int Mp, Np;            // padded rows of the slice stacks (multiples of BM / BN)
    int ns;                // slices
    int symmetric;         // 1: only tiles touching the upper triangle are computed, only elements n >= m are written
    const int* Ea; const int* Eb;   // per-row exponents
    double* C; long ldc;   // fp64 output, row-major [M, ldc]
    // optional transposed-scatter epilogue (stage 1 of DF-K): C element (m, n) is stored at
    //   C[(m % inner) * ldc + (m / inner) * N + n]   when inner > 0
    int inner;
    int a_row0;            // first row of the A stack used by this GEMM (row blocks of a persistent stack)
    // work item = (tile, K range); ksplit K ranges of kb_per K blocks per tile, ntiles tiles.  Partial results of the K ranges
    // meet in fp64 reductions (accumulate)
    int ksplit, kb_per, ntiles, accumulate;
    // stage 1: optional per-output-row maxima (bit pattern of max |C| per row m % inner, 64-bit atomicMax), so that the slicing
    // of Y needs no row-maximum pass of its own
    unsigned long long* rowmax;
    // stage 1 writing the int8 slices of Y itself (no fp64 Y): yq = base of the Y stack [ns][y_Rp][y_Kp], row = m % inner,
    // column = (m / inner) * y_ncolp + n (y_ncolp = N padded to 16), Ey[row] = exponent BOUND of the row (known before the GEMM:
    // Cauchy-Schwarz on the row norms of the tensor block and the column norms of the right factor)
    int8_t* yq; const int* Ey; int y_Rp, y_Kp, y_ncolp;
};

// ---------------------------------------------------------------------------------------------- PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity)
{
    uint32_t ok;
    do {
        asm volatile(
            "{\n\t"
            ".reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t"
            "}\n"
            : "=r"(ok)
            : "r"(smem_u32(bar)), "r"(parity)
            : "memory");
    } while (!ok);
}
// 2^e for -1022 <= e <= 1023 only (outside, the bit pattern wraps into a wrong value of either sign)
__device__ __forceinline__ double pow2i(int e) { return __longlong_as_double((long long)(e + 1023) << 52); }
// x 2^e with one rounding for every int e: one multiply in the range of pow2i, ldexp beyond it, so that a product of two tiny
// (or huge) row exponents underflows to a subnormal / 0 (overflows to inf) instead of taking the wrapped value of pow2i
__device__ __forceinline__ double scale2(double x, int e) { return (e >= -1022 && e <= 1023) ? x * pow2i(e) : ldexp(x, e); }
// the two factors s1 s2 = 2^e, e <= 2046, of a scaling UP that may leave the range of pow2i: x s1 is exact (s1 = 1 unless
// e > 1023, and then |x| < 2^-975 is lifted into the normal range), so fma(x * s1, s2, c) rounds once, like fma(x, 2^e, c)
__device__ __forceinline__ void pow2_split(int e, double& s1, double& s2)
{
    const int e1 = e > 1023 ? e - 1023 : 0;
    s1 = pow2i(e1); s2 = pow2i(e - e1);
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* tmap, uint64_t* bar, int c0, int c1)
{
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 ::"r"(smem_u32(smem_dst)), "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
                 : "memory");
}
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* tmap)
{
    asm volatile("prefetch.tensormap [%0];" ::"l"(tmap) : "memory");
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// d[64 x N] += A[64 x 32] * B[N x 32]^T, s8 x s8 -> s32, both operands K-major in shared memory.
// Fragment of thread t of the warpgroup: d[4j + 2i + c] = D[16 (t/32) + (t%32)/4 + 8i][8j + 2(t%4) + c], j < N/8.
template <int N>
__device__ __forceinline__ void wgmma_s8(int32_t* d, uint64_t desc_a, uint64_t desc_b);
template <> __device__ __forceinline__ void wgmma_s8<32>(int32_t* d, uint64_t desc_a, uint64_t desc_b)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\twgmma.mma_async.sync.aligned.m64n32k32.s32.s8.s8 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p;\n\t}\n"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15])
                 : "l"(desc_a), "l"(desc_b), "r"(1));
}
template <> __device__ __forceinline__ void wgmma_s8<64>(int32_t* d, uint64_t desc_a, uint64_t desc_b)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\twgmma.mma_async.sync.aligned.m64n64k32.s32.s8.s8 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p;\n\t}\n"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31])
                 : "l"(desc_a), "l"(desc_b), "r"(1));
}
template <> __device__ __forceinline__ void wgmma_s8<96>(int32_t* d, uint64_t desc_a, uint64_t desc_b)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %50, 0;\n\twgmma.mma_async.sync.aligned.m64n96k32.s32.s8.s8 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, %48, %49, p;\n\t}\n"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47])
                 : "l"(desc_a), "l"(desc_b), "r"(1));
}
template <> __device__ __forceinline__ void wgmma_s8<128>(int32_t* d, uint64_t desc_a, uint64_t desc_b)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\twgmma.mma_async.sync.aligned.m64n128k32.s32.s8.s8 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p;\n\t}\n"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
                 : "l"(desc_a), "l"(desc_b), "r"(1));
}
template <> __device__ __forceinline__ void wgmma_s8<160>(int32_t* d, uint64_t desc_a, uint64_t desc_b)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %82, 0;\n\twgmma.mma_async.sync.aligned.m64n160k32.s32.s8.s8 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79}, %80, %81, p;\n\t}\n"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63]), "+r"(d[64]), "+r"(d[65]), "+r"(d[66]), "+r"(d[67]), "+r"(d[68]), "+r"(d[69]), "+r"(d[70]), "+r"(d[71]), "+r"(d[72]), "+r"(d[73]), "+r"(d[74]), "+r"(d[75]), "+r"(d[76]), "+r"(d[77]), "+r"(d[78]), "+r"(d[79])
                 : "l"(desc_a), "l"(desc_b), "r"(1));
}
template <> __device__ __forceinline__ void wgmma_s8<192>(int32_t* d, uint64_t desc_a, uint64_t desc_b)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %98, 0;\n\twgmma.mma_async.sync.aligned.m64n192k32.s32.s8.s8 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95}, %96, %97, p;\n\t}\n"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63]), "+r"(d[64]), "+r"(d[65]), "+r"(d[66]), "+r"(d[67]), "+r"(d[68]), "+r"(d[69]), "+r"(d[70]), "+r"(d[71]), "+r"(d[72]), "+r"(d[73]), "+r"(d[74]), "+r"(d[75]), "+r"(d[76]), "+r"(d[77]), "+r"(d[78]), "+r"(d[79]), "+r"(d[80]), "+r"(d[81]), "+r"(d[82]), "+r"(d[83]), "+r"(d[84]), "+r"(d[85]), "+r"(d[86]), "+r"(d[87]), "+r"(d[88]), "+r"(d[89]), "+r"(d[90]), "+r"(d[91]), "+r"(d[92]), "+r"(d[93]), "+r"(d[94]), "+r"(d[95])
                 : "l"(desc_a), "l"(desc_b), "r"(1));
}
template <> __device__ __forceinline__ void wgmma_s8<224>(int32_t* d, uint64_t desc_a, uint64_t desc_b)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %114, 0;\n\twgmma.mma_async.sync.aligned.m64n224k32.s32.s8.s8 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111}, %112, %113, p;\n\t}\n"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63]), "+r"(d[64]), "+r"(d[65]), "+r"(d[66]), "+r"(d[67]), "+r"(d[68]), "+r"(d[69]), "+r"(d[70]), "+r"(d[71]), "+r"(d[72]), "+r"(d[73]), "+r"(d[74]), "+r"(d[75]), "+r"(d[76]), "+r"(d[77]), "+r"(d[78]), "+r"(d[79]), "+r"(d[80]), "+r"(d[81]), "+r"(d[82]), "+r"(d[83]), "+r"(d[84]), "+r"(d[85]), "+r"(d[86]), "+r"(d[87]), "+r"(d[88]), "+r"(d[89]), "+r"(d[90]), "+r"(d[91]), "+r"(d[92]), "+r"(d[93]), "+r"(d[94]), "+r"(d[95]), "+r"(d[96]), "+r"(d[97]), "+r"(d[98]), "+r"(d[99]), "+r"(d[100]), "+r"(d[101]), "+r"(d[102]), "+r"(d[103]), "+r"(d[104]), "+r"(d[105]), "+r"(d[106]), "+r"(d[107]), "+r"(d[108]), "+r"(d[109]), "+r"(d[110]), "+r"(d[111])
                 : "l"(desc_a), "l"(desc_b), "r"(1));
}
template <> __device__ __forceinline__ void wgmma_s8<256>(int32_t* d, uint64_t desc_a, uint64_t desc_b)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\twgmma.mma_async.sync.aligned.m64n256k32.s32.s8.s8 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p;\n\t}\n"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63]), "+r"(d[64]), "+r"(d[65]), "+r"(d[66]), "+r"(d[67]), "+r"(d[68]), "+r"(d[69]), "+r"(d[70]), "+r"(d[71]), "+r"(d[72]), "+r"(d[73]), "+r"(d[74]), "+r"(d[75]), "+r"(d[76]), "+r"(d[77]), "+r"(d[78]), "+r"(d[79]), "+r"(d[80]), "+r"(d[81]), "+r"(d[82]), "+r"(d[83]), "+r"(d[84]), "+r"(d[85]), "+r"(d[86]), "+r"(d[87]), "+r"(d[88]), "+r"(d[89]), "+r"(d[90]), "+r"(d[91]), "+r"(d[92]), "+r"(d[93]), "+r"(d[94]), "+r"(d[95]), "+r"(d[96]), "+r"(d[97]), "+r"(d[98]), "+r"(d[99]), "+r"(d[100]), "+r"(d[101]), "+r"(d[102]), "+r"(d[103]), "+r"(d[104]), "+r"(d[105]), "+r"(d[106]), "+r"(d[107]), "+r"(d[108]), "+r"(d[109]), "+r"(d[110]), "+r"(d[111]), "+r"(d[112]), "+r"(d[113]), "+r"(d[114]), "+r"(d[115]), "+r"(d[116]), "+r"(d[117]), "+r"(d[118]), "+r"(d[119]), "+r"(d[120]), "+r"(d[121]), "+r"(d[122]), "+r"(d[123]), "+r"(d[124]), "+r"(d[125]), "+r"(d[126]), "+r"(d[127])
                 : "l"(desc_a), "l"(desc_b), "r"(1));
}

// exact int32 -> fp64 on the FP64 add pipe (one LOP + one DADD instead of a conversion instruction):
// the double with high word 0x43300000 and low word (x ^ 2^31) is 2^52 + 2^31 + x
__device__ __forceinline__ double i2d_exact(uint32_t x)
{
    return __hiloint2double(0x43300000, (int)(x ^ 0x80000000u)) - 4503601774854144.0;
}

// K-major, 128B-swizzled shared-memory matrix descriptor of wgmma:
// start>>4 [0,14) | LBO>>4 [16,30) (unused for swizzled K-major, canonical 1) | SBO>>4 [32,46): 8 rows x 128 B between
// row groups | layout type [62,64): 1 = SWIZZLE_128B.  The tile base is 1024-byte aligned; the K offset inside the swizzle
// row is added to the start address.
__device__ __forceinline__ uint64_t make_desc_k_sw128(uint32_t smem_addr)
{
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(1024 >> 4) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}

// work item -> (m tile, n tile, K-block range).  Items are numbered K range slowest, tile fastest (CTAs running side by side
// share the A tile of their m tile in L2); symmetric: only the tiles with (nt + 1) * BN > mt * BM, i.e. nt >= 2 mt.
__device__ __forceinline__ void decode_item(const GemmParams& P, int item, int ntn, int nkb, int& mt, int& nt, int& kb0, int& kb1)
{
    const int ks = item / P.ntiles;
    int tile = item - ks * P.ntiles;
    if (P.symmetric) {
        mt = 0;
        for (;;) {
            const int cnt = ntn - (BM / BN) * mt;
            if (tile < cnt) break;
            tile -= cnt; mt++;
        }
        nt = (BM / BN) * mt + tile;
    } else {
        mt = tile / ntn; nt = tile - mt * ntn;
    }
    kb0 = ks * P.kb_per;
    kb1 = (kb0 + P.kb_per < nkb) ? kb0 + P.kb_per : nkb;
}

// ---------------------------------------------------------------------------------------------- GEMM kernel
// One K block of a consumer warpgroup, A slices k = K .. NS-1 (compile-time k and l: straight-line code).  A_k (64 rows of this
// warpgroup) times each B slice l = 0 .. NS-1-k: one m64n32k32 wgmma per pair and 32 bytes of K into the accumulator of group
// k + l (acc[16 (k + l)] .. +15).  Every wgmma has the same shape and writes one whole, disjoint 16-register block, so ptxas
// keeps them in flight (mixed shapes over overlapping sub-ranges of acc serialise the wgmma pipeline).  The A stage of slice
// k-1 is handed back as soon as the products of slice k are issued behind it.
template <int NS, int K>
struct SliceMMA {
    static __device__ __forceinline__ void run(int32_t* acc, uint8_t* sA, uint64_t* afull, uint64_t* aempty, uint32_t b0, int h,
                                               int lane, int& sa, uint32_t& pa, int prev)
    {
        mbar_wait(&afull[sa], pa);
        const uint32_t a0 = smem_u32(sA + sa * A_STAGE_BYTES + h * (BM / 2) * BK);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < BK / UK; kk++)
#pragma unroll
            for (int l = 0; l < NS - K; l++)
                wgmma_s8<BN>(acc + (BN / 2) * (K + l), make_desc_k_sw128(a0 + kk * UK), make_desc_k_sw128(b0 + l * B_SLICE_BYTES + kk * UK));
        wgmma_commit();
        wgmma_wait<1>();
        if (K > 0 && lane == 0) mbar_arrive(&aempty[prev]);
        const int cur = sa;
        if (++sa == NSA) { sa = 0; pa ^= 1; }
        SliceMMA<NS, K + 1>::run(acc, sA, afull, aempty, b0, h, lane, sa, pa, cur);
    }
};
template <int NS>
struct SliceMMA<NS, NS> {
    static __device__ __forceinline__ void run(int32_t*, uint8_t*, uint64_t*, uint64_t* aempty, uint32_t, int, int lane, int&,
                                               uint32_t&, int prev)
    {
        wgmma_wait<0>();
        if (lane == 0) mbar_arrive(&aempty[prev]);
    }
};

// tmapA / tmapB: 2-D uint8 tensors [ns*Mp (resp. ns*Np) rows][Kp bytes], box {BK, BM} / {BK, BN}, SWIZZLE_128B.
// Persistent: CTA b takes the work items b, b + gridDim.x, ...  Per K block of an item the producer loads the NS slices of the
// B tile once (back to back: rows l*BN of the stage form one K-major operand of NS*BN rows) and the NS slice tiles A_k one after
// the other; all NS(NS+1)/2 slice products of the K block are formed from these loads (A-stationary: no operand is re-read).
// The epilogue is one of
//   yq:         the int8 slices of Y are cut from the fp64 tile (stage 1 of DF-K, Y never exists in fp64),
//   accumulate: fp64 reductions into C (stage 2 of DF-K, K ranges of one tile meet there),
//   otherwise:  plain stores into C (+ row maxima).
template <int NS>
__global__ void __launch_bounds__(NTHREADS, 1)
i8gemm_kernel(const __grid_constant__ CUtensorMap tmapA, const __grid_constant__ CUtensorMap tmapB, const GemmParams P)
{
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // 1024-byte aligned, still known to be shared memory
    constexpr int B_STAGE_BYTES = NS * B_SLICE_BYTES;
    uint8_t* sA = smem;
    uint8_t* sB = smem + NSA * A_STAGE_BYTES;
    uint64_t* afull = (uint64_t*)(sB + NSB * B_STAGE_BYTES);   // [NSA] operands landed (TMA -> wgmma)
    uint64_t* aempty = afull + NSA;                              // [NSA] stage consumed (wgmma -> TMA), one arrival per consumer warp
    uint64_t* bfull = aempty + NSA;                              // [NSB]
    uint64_t* bempty = bfull + NSB;                              // [NSB]

    const int wg = threadIdx.x >> 7, lane = threadIdx.x & 31;
    const int nkb = P.Kp / BK;
    const int ntn = (P.N + BN - 1) / BN;
    const int nitems = P.ntiles * P.ksplit;

    if (threadIdx.x == 0) {
        prefetch_tmap(&tmapA);
        prefetch_tmap(&tmapB);
        for (int i = 0; i < NSA; i++) { mbar_init(&afull[i], 1); mbar_init(&aempty[i], NCONSUMER_WARPS); }
        for (int i = 0; i < NSB; i++) { mbar_init(&bfull[i], 1); mbar_init(&bempty[i], NCONSUMER_WARPS); }
        fence_barrier_init();
    }
    __syncthreads();

    if (wg == 0) {
        // ===== TMA producer: hands its registers to the consumers (128 x 40 + 256 x 232 <= 64 K) =====
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
        if (threadIdx.x == 0) {
            int sa = 0, sb = 0; uint32_t pa = 0, pb = 0;
            for (int item = blockIdx.x; item < nitems; item += gridDim.x) {
                int mt, nt, kb0, kb1;
                decode_item(P, item, ntn, nkb, mt, nt, kb0, kb1);
                for (int kb = kb0; kb < kb1; kb++) {
                    mbar_wait(&bempty[sb], pb ^ 1);
                    mbar_expect_tx(&bfull[sb], B_STAGE_BYTES);
                    for (int l = 0; l < NS; l++)
                        tma_load_2d(sB + sb * B_STAGE_BYTES + l * B_SLICE_BYTES, &tmapB, &bfull[sb], kb * BK, l * P.Np + nt * BN);
                    if (++sb == NSB) { sb = 0; pb ^= 1; }
                    for (int k = 0; k < NS; k++) {
                        mbar_wait(&aempty[sa], pa ^ 1);
                        mbar_expect_tx(&afull[sa], A_STAGE_BYTES);
                        tma_load_2d(sA + sa * A_STAGE_BYTES, &tmapA, &afull[sa], kb * BK, k * P.Mp + P.a_row0 + mt * BM);
                        if (++sa == NSA) { sa = 0; pa ^= 1; }
                    }
                }
            }
        }
        return;
    }

    // ===== consumers: warpgroup h = wg - 1 owns rows 64 h .. 64 h + 63 of the tile; 16 NS accumulator registers per thread =====
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
    const int h = wg - 1;
    const int t = threadIdx.x & 127;
    const int rq = 16 * (t >> 5) + (lane >> 2);     // fragment rows rq, rq + 8 of this warpgroup's 64
    const int cq = 2 * (lane & 3);                  // fragment columns 8j + cq, 8j + cq + 1
    constexpr int NF = BN / 2;                      // accumulator registers per group
    int sa = 0, sb = 0; uint32_t pa = 0, pb = 0;
    for (int item = blockIdx.x; item < nitems; item += gridDim.x) {
        int mt, nt, kb0, kb1;
        decode_item(P, item, ntn, nkb, mt, nt, kb0, kb1);
        int32_t acc[NS * NF];
#pragma unroll
        for (int j = 0; j < NS * NF; j++) acc[j] = 0;
        for (int kb = kb0; kb < kb1; kb++) {
            mbar_wait(&bfull[sb], pb);
            SliceMMA<NS, 0>::run(acc, sA, afull, aempty, smem_u32(sB + sb * B_STAGE_BYTES), h, lane, sa, pa, 0);
            if (lane == 0) mbar_arrive(&bempty[sb]);
            if (++sb == NSB) { sb = 0; pb ^= 1; }
        }
        double accv[NF];
#pragma unroll
        for (int j = 0; j < NF; j++) accv[j] = 0.0;
#pragma unroll
        for (int g = NS - 1; g >= 0; g--) {
            const double w = pow2i(-12 - 7 * g);
#pragma unroll
            for (int j = 0; j < NF; j++) accv[j] += i2d_exact((uint32_t)acc[g * NF + j]) * w;
        }

        const int nb = nt * BN;
#pragma unroll
        for (int i = 0; i < 2; i++) {
            const int m = mt * BM + h * (BM / 2) + rq + 8 * i;
            if (m >= P.M) continue;
            const int ea = __ldg(P.Ea + P.a_row0 + m);
            if (P.yq) {
                // Y never exists in fp64: scale the row by its exponent bound and cut the balanced 7-bit digits here
                // (round-to-nearest by the 1.5*2^52 trick: two adds per digit instead of a rounding and a conversion instruction)
                const int yrow = m % P.inner;
                const long ycol0 = (long)(m / P.inner) * P.y_ncolp;
                const int esc = ea + 6 - __ldg(P.Ey + yrow);
                int8_t* dst0 = P.yq + (long)yrow * P.y_Kp + ycol0;
                const long sstride = (long)P.y_Rp * P.y_Kp;
#pragma unroll
                for (int j = 0; j < BN / 8; j++) {
                    const int n = nb + 8 * j + cq;
                    if (n >= P.y_ncolp) continue;    // y_ncolp is a multiple of 16: both columns of the pair are inside
                    double r0 = scale2(accv[4 * j + 2 * i], esc + __ldg(P.Eb + n));
                    double r1 = scale2(accv[4 * j + 2 * i + 1], esc + __ldg(P.Eb + n + 1));
                    for (int s_ = 0; s_ < NS; s_++) {
                        const double t0 = r0 + 6755399441055744.0, t1 = r1 + 6755399441055744.0;
                        const double q0 = t0 - 6755399441055744.0, q1 = t1 - 6755399441055744.0;
                        const unsigned short pk = (unsigned short)(((unsigned)__double2loint(t0) & 255u) | (((unsigned)__double2loint(t1) & 255u) << 8));
                        *reinterpret_cast<unsigned short*>(dst0 + s_ * sstride + n) = pk;
                        r0 = (r0 - q0) * 128.0; r1 = (r1 - q1) * 128.0;
                    }
                }
                continue;
            }
            const long off = (P.inner > 0) ? (long)(m % P.inner) * P.ldc + (long)(m / P.inner) * P.N : (long)m * P.ldc;
            double* dst = P.C + off;
            if (P.accumulate) {
#pragma unroll
                for (int j = 0; j < BN / 8; j++)
#pragma unroll
                    for (int c = 0; c < 2; c++) {
                        const int n = nb + 8 * j + cq + c;
                        if (n < P.N && (!P.symmetric || n >= m)) atomicAdd(dst + n, scale2(accv[4 * j + 2 * i + c], ea + __ldg(P.Eb + n)));
                    }
                continue;
            }
            double vmax = 0.0;
#pragma unroll
            for (int j = 0; j < BN / 8; j++) {
                const int n = nb + 8 * j + cq;
                if (n + 1 < P.N && ((off + n) & 1) == 0) {
                    // both columns inside and 16-byte aligned: one 128-bit store
                    const double v0 = scale2(accv[4 * j + 2 * i], ea + __ldg(P.Eb + n));
                    const double v1 = scale2(accv[4 * j + 2 * i + 1], ea + __ldg(P.Eb + n + 1));
                    *reinterpret_cast<double2*>(dst + n) = make_double2(v0, v1);
                    vmax = fmax(vmax, fmax(fabs(v0), fabs(v1)));
                } else {
#pragma unroll
                    for (int c = 0; c < 2; c++)
                        if (n + c < P.N) {
                            const double v = scale2(accv[4 * j + 2 * i + c], ea + __ldg(P.Eb + n + c));
                            dst[n + c] = v;
                            vmax = fmax(vmax, fabs(v));
                        }
                }
            }
            if (P.rowmax && vmax > 0.0)
                atomicMax(P.rowmax + (P.inner > 0 ? m % P.inner : m), (unsigned long long)__double_as_longlong(vmax));
        }
    }
}

// ---------------------------------------------------------------------------------------------- slicing kernels
// X: [R, K] fp64 row-major (row stride ldx).  out: [ns][Rp][Kp] int8, rows written at out_row0 + r; E[out_row0 + r].
// Pad rows / pad columns of the stack must be zero (stack_alloc memsets once; pad columns are rewritten here).
// (1) one warp per row: many short rows (the unpacked tensor: K = nao).
__global__ void __launch_bounds__(256) split_rows_kernel(const double* __restrict__ X, long ldx, int R, int K, int Rp, int Kp, int ns,
                                                         int out_row0, int8_t* __restrict__ out, int* __restrict__ E)
{
    const int r = blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (r >= R) return;
    const double* x = X + (long)r * ldx;
    double mx = 0.0;
    for (int k = lane; k < K; k += 32) mx = fmax(mx, fabs(x[k]));
    for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    int e = 0;
    if (mx > 0.0) { frexp(mx, &e); }         // mx = f * 2^e, f in [0.5,1)  =>  |x| / 2^e < 1
    if (lane == 0) E[out_row0 + r] = e;
    for (int k = lane; k < Kp; k += 32) {
        double rr = (k < K) ? scale2(x[k], 6 - e) : 0.0;     // 2^(6-e) alone overflows for a subnormal row maximum
        for (int s = 0; s < ns; s++) {
            double qv = rint(rr);
            out[((long)s * Rp + out_row0 + r) * Kp + k] = (int8_t)(int)qv;
            rr = (rr - qv) * 128.0;
        }
    }
}
// (2) few long rows (Y: K = naux_block * nocc): grid (segments, rows); row maxima through 64-bit atomicMax on |x| bits
__global__ void __launch_bounds__(256) rowmax_kernel(const double* __restrict__ X, long ldx, int K, long seglen,
                                                     unsigned long long* __restrict__ maxbits)
{
    const int r = blockIdx.y;
    const long k0 = blockIdx.x * seglen, k1 = (k0 + seglen < K) ? k0 + seglen : K;
    const double* x = X + (long)r * ldx;
    double mx = 0.0;
    for (long k = k0 + threadIdx.x; k < k1; k += 256) mx = fmax(mx, fabs(x[k]));
    for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if ((threadIdx.x & 31) == 0 && mx > 0.0) atomicMax(&maxbits[r], (unsigned long long)__double_as_longlong(mx));
}
__global__ void __launch_bounds__(256) split_long_kernel(const double* __restrict__ X, long ldx, int K, int Rp, int Kp, int ns, long seglen,
                                                         const unsigned long long* __restrict__ maxbits, int8_t* __restrict__ out,
                                                         int* __restrict__ E)
{
    const int r = blockIdx.y;
    const long k0 = blockIdx.x * seglen, k1 = (k0 + seglen < Kp) ? k0 + seglen : Kp;
    const double* x = X + (long)r * ldx;
    const double mx = __longlong_as_double((long long)maxbits[r]);
    int e = 0;
    if (mx > 0.0) { frexp(mx, &e); }
    if (blockIdx.x == 0 && threadIdx.x == 0) E[r] = e;
    // 8 consecutive elements per thread: one 64-bit store per slice (a warp writes 256 contiguous bytes per instruction);
    // k0, k1 and Kp are multiples of 8 (segments of 8192, Kp multiple of 128)
    for (long k = k0 + threadIdx.x * 8L; k < k1; k += 256 * 8L) {
        double rr[8];
#pragma unroll
        for (int j = 0; j < 8; j++) rr[j] = (k + j < K) ? scale2(x[k + j], 6 - e) : 0.0;
        for (int s = 0; s < ns; s++) {
            unsigned long long pack = 0;
#pragma unroll
            for (int j = 0; j < 8; j++) {
                const double qv = rint(rr[j]);
                pack |= (unsigned long long)(unsigned char)(int8_t)(int)qv << (8 * j);
                rr[j] = (rr[j] - qv) * 128.0;
            }
            *reinterpret_cast<unsigned long long*>(out + ((long)s * Rp + r) * Kp + k) = pack;
        }
    }
}


// (3) the DF tensor, straight from its PACKED rows (reference layout cderi[P][a(a+1)/2 + b], a >= b, pyscf/df/incore.py:134-136)
//     to the int8 slices of the UNPACKED matrices A_P[a][b] = A_P[b][a] that stage 1 of DF-K multiplies: no fp64 unpacked
//     copy is ever written.  Row (P, a) of the stack is scaled by its own exponent (max over the whole unpacked row).
constexpr int EXP_NONE = (int)0x80808080;    // "no non-zero element seen yet" (byte pattern of a memset with 0x80)
__device__ __forceinline__ int frexp_exp(double v)   // e with |v| = f 2^e, f in [0.5, 1); v != 0
{
    return (int)((__double_as_longlong(v) >> 52) & 0x7ff) - 1022;
}
// rowexp[P][a] = exponent of max_b |A_P[a][b]|, accumulated with integer atomicMax; the caller fills rowexp with EXP_NONE.
// grid (ceil(nao / 64), nr): a CTA reads the packed rows a0 .. a0+63 of auxiliary row P once, coalesced; an element (a, b)
// counts for row a (warp reduction) and for row b (shared-memory atomicMax, flushed once per CTA).
// rownorm2[P][a] (optional, zeroed by the caller) = sum_b A_P[a][b]^2 in single precision: the row norms behind the exponent
// bound of Y when stage 1 cuts the slices of Y itself.
// Pair-screened rows (MAP): a row of length npair holds only the kept packed columns; element t of the packed triangle is
// row[col_of[t]], or 0 for col_of[t] < 0.  On the same values both variants give the same exponents, norms and digits.
template <bool MAP>
__device__ __forceinline__ double packed_load(const double* __restrict__ row, const int* __restrict__ col_of, long t)
{
    if constexpr (MAP) {
        const int c = col_of[t];
        return c >= 0 ? row[c] : 0.0;
    } else {
        return row[t];
    }
}
template <bool MAP>
__global__ void __launch_bounds__(256) packed_rowexp_kernel(const double* __restrict__ cderi, long npair, int nao, int* __restrict__ rowexp,
                                                            float* __restrict__ rownorm2, const int* __restrict__ col_of)
{
    extern __shared__ int emax_s[];          // [nao] exponents, then [nao] partial squared norms
    float* ss = reinterpret_cast<float*>(emax_s + nao);
    const int P = blockIdx.y;
    const double* row = cderi + (long)P * npair;
    const int a0 = blockIdx.x * 64, a1 = (a0 + 64 < nao) ? a0 + 64 : nao;
    for (int b = threadIdx.x; b < a1; b += 256) { emax_s[b] = EXP_NONE; ss[b] = 0.0f; }
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int a = a0 + warp; a < a1; a += 8) {
        const long ta = (long)a * (a + 1) / 2;
        int em = EXP_NONE;
        float sq = 0.0f;
        for (int b = lane; b <= a; b += 32) {
            const double v = fabs(packed_load<MAP>(row, col_of, ta + b));
            if (v > 0.0) {
                const int e = frexp_exp(v);
                em = e > em ? e : em;
                if (e > emax_s[b]) atomicMax(&emax_s[b], e);
                const float v2 = (float)(v * v);
                sq += v2;
                if (rownorm2 && b < a) atomicAdd(&ss[b], v2);      // the element also belongs to row b of the symmetric matrix
            }
        }
        for (int o = 16; o > 0; o >>= 1) {
            const int t = __shfl_xor_sync(0xffffffffu, em, o); em = t > em ? t : em;
            sq += __shfl_xor_sync(0xffffffffu, sq, o);
        }
        if (lane == 0 && em != EXP_NONE) {
            atomicMax(&rowexp[(long)P * nao + a], em);
            if (rownorm2) atomicAdd(&rownorm2[(long)P * nao + a], sq);
        }
    }
    __syncthreads();
    for (int b = threadIdx.x; b < a1; b += 256)
        if (emax_s[b] != EXP_NONE) {
            atomicMax(&rowexp[(long)P * nao + b], emax_s[b]);
            if (rownorm2 && ss[b] > 0.0f) atomicAdd(&rownorm2[(long)P * nao + b], ss[b]);
        }
}

// Exponent bound of the rows of Y = A_P C~ over a block of nr auxiliary rows, before the GEMM (Cauchy-Schwarz):
//   |Y[nu,(P,i)]| <= ||A_P[nu,:]||_2 * max_i ||C~[:,i]||_2      Ey[nu] = exponent of 1.001 * max_P ... (|y| < 2^Ey)
// cmax2: device scalar, max_i sum_mu C~[mu,i]^2 (colnorm_max_kernel).  One thread per nu.
__global__ void yexp_bound_kernel(const float* __restrict__ rownorm2, int nr, int nao, const double* __restrict__ cmax2, int* __restrict__ Ey)
{
    const int nu = blockIdx.x * blockDim.x + threadIdx.x;
    if (nu >= nao) return;
    float m = 0.0f;
    for (int P = 0; P < nr; P++) m = fmaxf(m, rownorm2[(long)P * nao + nu]);
    const double bound = 1.001 * sqrt((double)m * 1.0001 * cmax2[0]);
    Ey[nu] = bound > 0.0 ? frexp_exp(bound) : 0;
}
// cmax2[0] = max over the rows i of X[nrows][k] (row stride ldx) of sum_k X[i][k]^2; one warp per row; cmax2 zeroed by the caller
__global__ void __launch_bounds__(256) colnorm_max_kernel(const double* __restrict__ X, long ldx, int nrows, int k, unsigned long long* __restrict__ cmax2)
{
    const int r = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (r >= nrows) return;
    const double* x = X + (long)r * ldx;
    double sq = 0.0;
    for (int c = lane; c < k; c += 32) sq += x[c] * x[c];
    for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
    if (lane == 0 && sq > 0.0) atomicMax(cmax2, (unsigned long long)__double_as_longlong(sq));
}

constexpr int PT = 64;   // tile edge of split_packed_kernel
// grid (Kp/PT, Kp/PT, nr), CTAs with tile column > tile row leave at once.  CTA (ta, tb, P): loads the 64 x 64 tile
// A_P[ta*64 .., tb*64 ..] from the packed row (coalesced: 64 consecutive doubles per a), writes its slices to the rows
// (P, a) at columns b and — for off-diagonal tiles — the slices of the transposed tile to the rows (P, b) at columns a,
// four int8 per 32-bit store.  Columns nao..Kp-1 are written as zeros; pad ROWS of the stack are the caller's (memset).
// NS7: the slice count is the compile-time 7 (constant shift amounts, digits 3..6 from the low word, 0..1 from the high word)
// MAP: pair-screened rows read through col_of (packed_load)
template <bool NS7, bool MAP>
__global__ void __launch_bounds__(256) split_packed_kernel(const double* __restrict__ cderi, long npair, int nao,
                                                           const int* __restrict__ rowexp, int ns, int Rp, int Kp, int out_row0,
                                                           int8_t* __restrict__ out, int* __restrict__ E, const int* __restrict__ col_of)
{
    const int ta = blockIdx.x, tb = blockIdx.y, P = blockIdx.z;
    if (tb > ta) return;
    __shared__ double S[PT][PT + 1];
    const double* row = cderi + (long)P * npair;
    const int* ex = rowexp + (long)P * nao;
    const int t = threadIdx.x;
#pragma unroll 4
    for (int i = 0; i < PT * PT / 256; i++) {
        const int idx = t + 256 * i, al = idx >> 6, bl = idx & 63;
        const int a = ta * PT + al, b = tb * PT + bl;
        double v = 0.0;
        if (a < nao && b < nao) { const int hi = a > b ? a : b, lo = a > b ? b : a; v = packed_load<MAP>(row, col_of, (long)hi * (hi + 1) / 2 + lo); }
        S[al][bl] = v;
    }
    __syncthreads();
    const int c4 = (t & 15) * 4;     // four consecutive output columns per thread
    const long orow0 = (long)out_row0 + (long)P * nao;
#pragma unroll 1
    for (int pass = 0; pass < 2; pass++) {
        if (pass == 1 && ta == tb) break;
        const int trow = pass ? tb : ta, tcol = pass ? ta : tb;    // output rows / columns of this pass
#pragma unroll 1
        for (int i = 0; i < 4; i++) {
            const int rl = (t >> 4) + 16 * i;
            const int r = trow * PT + rl;
            if (r >= nao) continue;
            int e = ex[r];
            if (e == EXP_NONE) e = 0;
            if (tcol == 0 && c4 == 0) E[orow0 + r] = e;
            int8_t* dst = out + (orow0 + r) * Kp + tcol * PT + c4;
            if constexpr (NS7) {
                // N = rint(x 2^(48-e)), |N| <= 2^48, as (hi, lo) words of the mantissa of x*scale + 1.5*2^52 (offset 2^51 removed):
                // digit s sits at bit 7(6-s): s = 3..6 in lo[0,28), s = 2 across the words, s = 1 at hi[3,10), s = 0 = hi >> 10 (signed)
                double s1, scN;
                pow2_split(48 - e, s1, scN);
                unsigned lo[4]; int hi[4];
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    const double t_ = fma((pass ? S[c4 + j][rl] : S[rl][c4 + j]) * s1, scN, 6755399441055744.0);
                    lo[j] = (unsigned)__double2loint(t_);
                    hi[j] = (__double2hiint(t_) & 0x000FFFFF) - 0x00080000;     // remove exponent bits and the 2^51 offset
                }
                const long sstride = (long)Rp * Kp;
                unsigned pk[7];
#pragma unroll
                for (int s_ = 0; s_ < 7; s_++) pk[s_] = 0;
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    const unsigned l_ = lo[j];
                    const int h_ = hi[j];
                    pk[6] |= (l_ & 127u) << (8 * j);
                    pk[5] |= ((l_ >> 7) & 127u) << (8 * j);
                    pk[4] |= ((l_ >> 14) & 127u) << (8 * j);
                    pk[3] |= ((l_ >> 21) & 127u) << (8 * j);
                    pk[2] |= (__funnelshift_r(l_, (unsigned)h_, 28) & 127u) << (8 * j);
                    pk[1] |= (((unsigned)h_ >> 3) & 127u) << (8 * j);
                    pk[0] |= ((unsigned)(h_ >> 10) & 255u) << (8 * j);
                }
#pragma unroll
                for (int s_ = 0; s_ < 7; s_++) *reinterpret_cast<unsigned*>(dst + s_ * sstride) = pk[s_];
            } else if (ns <= 7) {
                // One FP64 operation per element instead of four per digit: N = rint(x 2^(6-e+7(ns-1))) (|N| < 2^48) sits in the
                // mantissa of x*scale + 1.5*2^52; its digits come out with integer shifts: the top one signed (-64..64), the others
                // 0..127 (two's-complement style, no carries).  Still an exact representation; the digit products of stage 1 are
                // bounded by 127*64 instead of 64*64, which the int32 accumulation bound covers up to K = nao < 37 000.
                double s1, scN;
                pow2_split(6 - e + 7 * (ns - 1), s1, scN);
                long long N[4];
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    const double t_ = fma((pass ? S[c4 + j][rl] : S[rl][c4 + j]) * s1, scN, 6755399441055744.0);
                    N[j] = (long long)(__double_as_longlong(t_) & 0x000FFFFFFFFFFFFFLL) - (1LL << 51);
                }
                for (int s_ = 0; s_ < ns; s_++) {
                    const int sh = 7 * (ns - 1 - s_);
                    unsigned pack = 0;
#pragma unroll
                    for (int j = 0; j < 4; j++) {
                        const int d_ = s_ == 0 ? (int)(N[j] >> sh) : (int)((N[j] >> sh) & 127);
                        pack |= (unsigned)(d_ & 0xff) << (8 * j);
                    }
                    *reinterpret_cast<unsigned*>(dst + (long)s_ * Rp * Kp) = pack;
                }
            } else {
                double s1, sc;
                pow2_split(6 - e, s1, sc);
                double rr[4];
#pragma unroll
                for (int j = 0; j < 4; j++) rr[j] = (pass ? S[c4 + j][rl] : S[rl][c4 + j]) * s1 * sc;
                for (int s_ = 0; s_ < ns; s_++) {
                    unsigned pack = 0;
#pragma unroll
                    for (int j = 0; j < 4; j++) {
                        const double qv = rint(rr[j]);
                        pack |= (unsigned)(unsigned char)(int8_t)(int)qv << (8 * j);
                        rr[j] = (rr[j] - qv) * 128.0;
                    }
                    *reinterpret_cast<unsigned*>(dst + (long)s_ * Rp * Kp) = pack;
                }
            }
        }
    }
}

}  // namespace i8g
}  // namespace b200jk
