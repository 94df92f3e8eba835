// Shared sm_90a building blocks: PTX wrappers for mbarrier / TMA / wgmma, the shared-memory matrix descriptors, the
// operand ring of the one-shot kernels (layout, barriers, the MMA warpgroup's K loop), the accumulator hand-over from
// the MMA warpgroup to the epilogue warps, and host-side tensor-map construction through the driver entry point (no
// libcuda link dependency), and the 128-pixel box plan of the TMA convolutions.  Included by gemm_tcgen05.cu,
// lstm_seq_tcgen05.cu, dcn_tcgen05.cu (the file names predate the Hopper port; nothing in them is tcgen05 any more) and
// conv_pingpong.cu.
#pragma once
#include "common.cuh"
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <type_traits>

namespace {
using namespace mr;
typedef __nv_bfloat16 bf16;

constexpr int BM = 128;
constexpr int BK = 64;             // 64 bf16 = 128 bytes = one swizzle atom
constexpr int WGMMA_K = 16;        // K depth of one wgmma instruction (16-bit operands)
constexpr int kMmaThreads = 128;    // one warpgroup

// ---------------------------------------------------------------- PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE;\n"
        "bra WAIT_LOOP;\n"
        "DONE:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void tma_load_2d(const CUtensorMap *map, uint64_t *bar, void *dst, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_load_4d(const CUtensorMap *map, uint64_t *bar, void *dst, int c0, int c1, int c2, int c3) {
    asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
                 ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
// shared -> global tensor store; completion is tracked per thread by bulk groups (commit, then wait)
__device__ __forceinline__ void tma_store_4d(const CUtensorMap *map, const void *src, int c0, int c1, int c2, int c3) {
    asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
                 ::"l"(map), "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// the stores committed before the last N groups have finished reading shared memory (their source may be overwritten)
template <int N> __device__ __forceinline__ void bulk_wait_group_read() {
    asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
// ... and have finished writing global memory
template <int N> __device__ __forceinline__ void bulk_wait_group() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }
// four 8x8 b16 matrices to shared memory: register i of every lane is matrix i's fragment in the mma accumulator layout
// (lane l holds row l / 4, columns 2 (l % 4), +1); lanes 8i..8i+7 give the addresses of matrix i's eight 16-byte rows
__device__ __forceinline__ void stmatrix_x4(uint32_t addr, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3) {
    asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(r0), "r"(r1), "r"(r2),
                 "r"(r3) : "memory");
}
// named barriers: `count` threads (whole warps) of the CTA; arrive does not wait
template <int COUNT> __device__ __forceinline__ void named_bar_sync(int id) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "n"(COUNT) : "memory");
}
template <int COUNT> __device__ __forceinline__ void named_bar_arrive(int id) {
    asm volatile("bar.arrive %0, %1;" ::"r"(id), "n"(COUNT) : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap *map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// register re-allocation between warpgroups (every warp of a warpgroup executes the same one)
template <int R> __device__ __forceinline__ void reg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R> __device__ __forceinline__ void reg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }

// ---------------------------------------------------------------- wgmma (one warpgroup = 128 threads issues it together)
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int PENDING> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(PENDING) : "memory"); }

// D[64 x N] (+)= A[64 x 16] * B[16 x N], 16-bit operands of element type E (bf16, the default, or __half) through
// shared-memory descriptors, fp32 accumulator fragment in registers.  TA / TB = 1: the operand is MN-major in shared memory
// (the instruction's transpose bits).
template <typename E> struct WgmmaElem;
template <> struct WgmmaElem<bf16> { static constexpr bool f16 = false; };
template <> struct WgmmaElem<__half> { static constexpr bool f16 = true; };
template <int N, typename E = bf16> struct Wgmma;
template <typename E> struct Wgmma<32, E> {
    template <int TA, int TB>
    static __device__ __forceinline__ void mma(float (&d)[16], uint64_t ad, uint64_t bd, uint32_t scale_d) {
#define MR_WGMMA_M64N32K16(AB) \
        asm volatile( \
            "{\n" \
            ".reg .pred p;\n" \
            "setp.ne.b32 p, %18, 0;\n" \
            "wgmma.mma_async.sync.aligned.m64n32k16.f32." AB "." AB " " \
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, " \
            "%16, %17, p, 1, 1, %19, %20;\n" \
            "}\n" \
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), \
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]) \
            : "l"(ad), "l"(bd), "r"(scale_d), "n"(TA), "n"(TB))
        if constexpr (WgmmaElem<E>::f16) MR_WGMMA_M64N32K16("f16");
        else MR_WGMMA_M64N32K16("bf16");
#undef MR_WGMMA_M64N32K16
    }
};
template <typename E> struct Wgmma<64, E> {
    template <int TA, int TB>
    static __device__ __forceinline__ void mma(float (&d)[32], uint64_t ad, uint64_t bd, uint32_t scale_d) {
#define MR_WGMMA_M64N64K16(AB) \
        asm volatile( \
            "{\n" \
            ".reg .pred p;\n" \
            "setp.ne.b32 p, %34, 0;\n" \
            "wgmma.mma_async.sync.aligned.m64n64k16.f32." AB "." AB " " \
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, " \
            "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, " \
            "%32, %33, p, 1, 1, %35, %36;\n" \
            "}\n" \
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), \
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), \
              "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), \
              "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]) \
            : "l"(ad), "l"(bd), "r"(scale_d), "n"(TA), "n"(TB))
        if constexpr (WgmmaElem<E>::f16) MR_WGMMA_M64N64K16("f16");
        else MR_WGMMA_M64N64K16("bf16");
#undef MR_WGMMA_M64N64K16
    }
};
template <typename E> struct Wgmma<128, E> {
    template <int TA, int TB>
    static __device__ __forceinline__ void mma(float (&d)[64], uint64_t ad, uint64_t bd, uint32_t scale_d) {
#define MR_WGMMA_M64N128K16(AB) \
        asm volatile( \
            "{\n" \
            ".reg .pred p;\n" \
            "setp.ne.b32 p, %66, 0;\n" \
            "wgmma.mma_async.sync.aligned.m64n128k16.f32." AB "." AB " " \
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, " \
            "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, " \
            "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, " \
            "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, " \
            "%64, %65, p, 1, 1, %67, %68;\n" \
            "}\n" \
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), \
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), \
              "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), \
              "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), \
              "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), \
              "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), \
              "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), \
              "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]) \
            : "l"(ad), "l"(bd), "r"(scale_d), "n"(TA), "n"(TB))
        if constexpr (WgmmaElem<E>::f16) MR_WGMMA_M64N128K16("f16");
        else MR_WGMMA_M64N128K16("bf16");
#undef MR_WGMMA_M64N128K16
    }
};
template <typename E> struct Wgmma<192, E> {
    template <int TA, int TB>
    static __device__ __forceinline__ void mma(float (&d)[96], uint64_t ad, uint64_t bd, uint32_t scale_d) {
#define MR_WGMMA_M64N192K16(AB) \
        asm volatile( \
            "{\n" \
            ".reg .pred p;\n" \
            "setp.ne.b32 p, %98, 0;\n" \
            "wgmma.mma_async.sync.aligned.m64n192k16.f32." AB "." AB " " \
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, " \
            "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, " \
            "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, " \
            "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, " \
            "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, " \
            "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95}, " \
            "%96, %97, p, 1, 1, %99, %100;\n" \
            "}\n" \
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), \
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), \
              "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), \
              "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), \
              "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), \
              "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), \
              "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), \
              "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), \
              "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), \
              "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), \
              "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), \
              "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]) \
            : "l"(ad), "l"(bd), "r"(scale_d), "n"(TA), "n"(TB))
        if constexpr (WgmmaElem<E>::f16) MR_WGMMA_M64N192K16("f16");
        else MR_WGMMA_M64N192K16("bf16");
#undef MR_WGMMA_M64N192K16
    }
};

// The 128 x BN fp32 accumulator of one MMA warpgroup: rows 0..63 in d[0], rows 64..127 in d[1] (two m64 instructions per
// 16-deep K step share the B descriptor).  When the K loop is over the warpgroup publishes it as a row-major shared
// memory tile [128][BN + 1] (odd pitch: a thread that owns a row reads consecutive columns without bank conflicts) that
// the epilogue warps read with acc_ld.
template <int BN> struct AccTile {
    static constexpr int LD = BN + 1;
    static constexpr int BYTES = BM * LD * 4;
    float d[2][BN / 2];
    template <int TA, int TB, typename E = bf16>
    __device__ __forceinline__ void mma(uint64_t a_lo, uint64_t a_hi, uint64_t b, uint32_t accumulate) {
        Wgmma<BN, E>::template mma<TA, TB>(d[0], a_lo, b, accumulate);
        Wgmma<BN, E>::template mma<TA, TB>(d[1], a_hi, b, accumulate);
    }
    // The same step as four 64-column instructions (b_lo / b_hi: the operand's two 64-column halves), for kernels whose
    // 768 threads leave too few registers per thread for the operands of one 128-column instruction.
    template <int TA, int TB, typename E = bf16>
    __device__ __forceinline__ void mma_halves(uint64_t a_lo, uint64_t a_hi, uint64_t b_lo, uint64_t b_hi, uint32_t accumulate) {
        static_assert(BN == 128, "two 64-column halves");
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            Wgmma<64, E>::template mma<TA, TB>(reinterpret_cast<float (&)[32]>(d[half][0]), half ? a_hi : a_lo, b_lo, accumulate);
            Wgmma<64, E>::template mma<TA, TB>(reinterpret_cast<float (&)[32]>(d[half][32]), half ? a_hi : a_lo, b_hi, accumulate);
        }
    }
    // fragment layout of wgmma m64nNk16: warp w of the warpgroup holds rows 16w..16w+15; d[4j + 2h + e] is row
    // 16w + lane / 4 + 8h, column 8j + 2 (lane % 4) + e
    __device__ __forceinline__ void store(float *tile, int wg_thread) const {
        const int w = wg_thread >> 5, l = wg_thread & 31;
#pragma unroll
        for (int half = 0; half < 2; ++half)
#pragma unroll
            for (int j = 0; j < BN / 8; ++j)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    float *dst = tile + (half * 64 + 16 * w + (l >> 2) + 8 * h) * LD + 8 * j + 2 * (l & 3);
                    dst[0] = d[half][4 * j + 2 * h];
                    dst[1] = d[half][4 * j + 2 * h + 1];
                }
    }
};
__device__ __forceinline__ void mma_group_sync() { asm volatile("bar.sync 15, 128;" ::: "memory"); }   // the MMA warpgroup only
// The calling warp's lane i reads NV consecutive columns of accumulator row (row0 + i) from the published tile.
template <int NV> __device__ __forceinline__ void acc_ld(const float *tile, int ld, int row0, int col0, uint32_t *r) {
    const float *src = tile + (row0 + (int)(threadIdx.x & 31)) * ld + col0;
#pragma unroll
    for (int j = 0; j < NV; ++j) r[j] = __float_as_uint(src[j]);
}
__device__ __forceinline__ bool elect_one() {
    uint32_t pred = 0;
    asm volatile(
        "{\n"
        ".reg .b32 rx;\n"
        ".reg .pred px;\n"
        "elect.sync rx|px, 0xffffffff;\n"
        "selp.u32 %0, 1, 0, px;\n"
        "}\n" : "=r"(pred));
    return pred != 0;
}

// shared-memory matrix descriptor, 128-byte swizzle (cute::GmmaDescriptor: start>>4 [0,14), LBO>>4 [16,30),
// SBO>>4 [32,46), layout_type=B128(1) [62,64))
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    return (uint64_t)((saddr >> 4) & 0x3FFF) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16) |
           ((uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32) | (1ull << 62);
}
// Descriptors of the 16-deep K step k of a 128-byte-swizzled operand tile at shared address `tile`; 8-row groups are
// 1024 B apart (SBO).  half = 1 addresses rows (or columns) 64.. of a 128-wide tile.
// K-major: 128-byte rows; the step starts 32 B further into the swizzle atom, the second half 64 rows * 128 B on.
__device__ __forceinline__ uint64_t desc_kmajor(uint32_t tile, int k, int half = 0) {
    return make_desc(tile + half * (64 * 128) + k * 32, 16, 1024);
}
// MN-major: 64-element MN atoms `atom` bytes apart (LBO); the step starts 16 K rows * 128 B on, the second half is the
// second atom.
__device__ __forceinline__ uint64_t desc_mnmajor(uint32_t tile, int k, uint32_t atom, int half = 0) {
    return make_desc(tile + half * atom + k * 2048, atom, 1024);
}

// ---------------------------------------------------------------- operand ring of the one-shot kernels
// STAGES x (A tile, B tile) from a 1024-byte aligned base, then the barriers full[STAGES], empty[STAGES], acc_full.
// When the K loop is over the accumulator tile is laid over the drained ring.
template <int BN, int STAGES_, int A_BYTES_ = BM * BK * 2, int B_BYTES_ = BN * BK * 2>
struct RingSmem {
    static constexpr int STAGES = STAGES_;
    static constexpr int A_BYTES = A_BYTES_;
    static constexpr int B_BYTES = B_BYTES_;
    static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
    static constexpr int BAR_OFF = STAGES * STAGE_BYTES;
    static constexpr int TOTAL = BAR_OFF + (2 * STAGES + 1) * 8 + 16 + 1024;   // + alignment slack
    static_assert(AccTile<BN>::BYTES <= BAR_OFF, "the accumulator tile is laid over the operand ring");
};

struct Ring {
    unsigned char *smem;        // the dynamic shared memory, 1024-byte aligned (the 128-byte swizzle needs it)
    uint64_t *full, *empty;     // [STAGES] each: stage loaded (TMA bytes + full_arrivals) / stage consumed (MMA warpgroup)
    uint64_t *acc_full;         // the accumulator tile is published
};
// Carves the barriers out at L::BAR_OFF (L: the layout, with STAGES and BAR_OFF) and initialises them; the one thread with
// init = true (warp 0, lane 0: the caller's own expression, which keeps the machine code of its kernel) first runs
// prefetch(), the tensor-map prefetches.  Every thread of the CTA must call it.
template <typename L, typename Prefetch>
__device__ __forceinline__ Ring ring_init(bool init, uint32_t full_arrivals, Prefetch prefetch) {
    constexpr int STAGES = L::STAGES;
    extern __shared__ unsigned char smem_raw[];
    Ring r;
    r.smem = (unsigned char *)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    r.full = (uint64_t *)(r.smem + L::BAR_OFF);
    r.empty = r.full + STAGES;
    r.acc_full = r.empty + STAGES;
    if (init) {
        prefetch();
        for (int s = 0; s < STAGES; ++s) { mbar_init(r.full + s, full_arrivals); mbar_init(r.empty + s, 1); }
        mbar_init(r.acc_full, 1);
        fence_barrier_init();
    }
    __syncthreads();
    return r;
}

// The MMA warpgroup's K loop over the ring: the wgmmas of block i are committed, then block i - 1 is known to have
// retired and its slot is handed back to the producers.  issue(i, s) queues the wgmmas of block i from stage s.
template <typename Issue>
__device__ __forceinline__ void mma_ring(int nkb, int stages, uint64_t *full, uint64_t *empty, bool leader, Issue issue) {
    uint64_t *pending = nullptr;
    for (int i = 0; i < nkb; ++i) {
        const int s = i % stages;
        mbar_wait(full + s, (i / stages) & 1);
        wgmma_fence();
        issue(i, s);
        wgmma_commit();
        wgmma_wait<1>();
        if (pending && leader) mbar_arrive(pending);
        pending = empty + s;
    }
    wgmma_wait<0>();
    if (pending && leader) mbar_arrive(pending);
}
// ... and the hand-over: the ring is drained (every load was consumed), so the accumulator tile is laid over it.
template <int BN>
__device__ __forceinline__ void mma_publish(const AccTile<BN> &acc, float *tile, uint64_t *acc_full, int mt) {
    mma_group_sync();
    acc.store(tile, mt);
    mma_group_sync();
    if (mt == 0) mbar_arrive(acc_full);
}


// ---------------------------------------------------------------- host: tensor maps through the driver entry point
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
    }
    return fn;
}

// 2-D bf16 tensor, `inner` contiguous elements per row, `outer` rows, row pitch ld elements; box {box_inner, box_outer}
int make_map(CUtensorMap *m, const void *base, int64_t inner, int64_t outer, int64_t ld, int box_inner, int box_outer) {
    EncodeTiledFn fn = encode_fn();
    if (!fn) { set_cuda_error(cudaErrorUnknown, "cuTensorMapEncodeTiled entry point"); return MR_ERR_CUDA; }
    cuuint64_t dims[2] = {(cuuint64_t)inner, (cuuint64_t)outer};
    cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
    cuuint32_t box[2] = {(cuuint32_t)box_inner, (cuuint32_t)box_outer};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void *>(base), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_cuda_error(cudaErrorInvalidValue, "cuTensorMapEncodeTiled"); return MR_ERR_CUDA; }
    return MR_OK;
}

// 4-D bf16 NHWC tensor map {C, W, H, N}, box {64, box_w, box_h, box_n}
// sw / sh > 1: strided traversal (every sw-th column, sh-th row) -- the box then spans box_w * sw columns of the tensor and
// delivers box_w of them (cuTensorMapEncodeTiled elementStrides)
// n_stride: elements from one image to the next (0: H * W * C, a dense tensor)
int make_map_nhwc(CUtensorMap *m, const void *base, int64_t C, int64_t W, int64_t H, int64_t N, int box_w, int box_h = 1,
                  int box_n = 1, int sw = 1, int sh = 1, int64_t n_stride = 0) {
    EncodeTiledFn fn = encode_fn();
    if (!fn) { set_cuda_error(cudaErrorUnknown, "cuTensorMapEncodeTiled entry point"); return MR_ERR_CUDA; }
    cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
    cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)(n_stride ? n_stride : H * W * C) * 2};
    cuuint32_t box[4] = {64, (cuuint32_t)(box_w * sw), (cuuint32_t)(box_h * sh), (cuuint32_t)box_n};
    cuuint32_t estr[4] = {1, (cuuint32_t)sw, (cuuint32_t)sh, 1};
    if (box[1] > 256 || box[2] > 256) { set_cuda_error(cudaErrorInvalidValue, "conv tensor map: strided box too large"); return MR_ERR_UNSUPPORTED; }
    CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void *>(base), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_cuda_error(cudaErrorInvalidValue, "cuTensorMapEncodeTiled(4d)"); return MR_ERR_CUDA; }
    return MR_OK;
}

// ---------------------------------------------------------------- 128-pixel output tiles of the TMA convolutions
// The output space [N, Ho, Wo] is tiled by boxes of bw x bh x bn = 128 pixels; the width is cut into segments of
// power-of-two widths (e.g. Wo = 65 -> one 64-wide segment + one 1-wide segment), each with its own activation tensor map.
// Tile row r of a box is pixel (n0 + r / (bw bh), h0 + r / bw % bh, w0 + r % bw): the row order of the TMA box itself.
constexpr int kMaxConvSegs = 4;
struct ConvSeg { int w0, bw, bh, bn, h_blocks, tile_begin; };

// Plans the segments of an [N, Ho, Wo] output over the activation x [N, H, W, C] (stride sw, sh) and encodes one tensor map
// per segment into tx.  *nseg = 0 when the plan needs more than kMaxConvSegs segments or a box the TMA cannot take;
// *tiles = the number of 128-pixel tiles of all segments.
int plan_conv_segments(const void *x, int N, int H, int W, int C, int Ho, int Wo, int sh, int sw, ConvSeg *seg,
                       CUtensorMap *tx, int *nseg, int *tiles) {
    *nseg = 0;
    *tiles = 0;
    int w0 = 0;
    while (w0 < Wo) {
        int bw = 128;
        while (bw > Wo - w0) bw >>= 1;
        const int nrep = (Wo - w0) / bw;                  /* consecutive segments of this width share geometry */
        int bh = 1;
        while (bh * 2 <= Ho && bw * bh * 2 <= 128) bh <<= 1;
        const int bn = 128 / (bw * bh);
        const int h_blocks = (int)ceil_div(Ho, bh), n_blocks = (int)ceil_div(N, bn);
        for (int rep = 0; rep < nrep; ++rep) {
            if (*nseg == kMaxConvSegs) { *nseg = 0; return MR_OK; }
            ConvSeg &sg = seg[*nseg];
            sg.w0 = w0; sg.bw = bw; sg.bh = bh; sg.bn = bn; sg.h_blocks = h_blocks; sg.tile_begin = *tiles;
            const int rc = make_map_nhwc(&tx[*nseg], x, C, W, H, N, bw, bh, bn, sw, sh);
            if (rc == MR_ERR_UNSUPPORTED) { *nseg = 0; return MR_OK; }
            if (rc) return rc;
            *tiles += h_blocks * n_blocks;
            ++*nseg;
            w0 += bw;
        }
    }
    return MR_OK;
}


}  // namespace
