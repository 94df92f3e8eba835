// Shared sm_90a building blocks: PTX wrappers for mbarrier / TMA / wgmma, the shared-memory matrix descriptor, the
// accumulator hand-over from the MMA warpgroup to the epilogue warps, MUFU-based activations, and host-side tensor-map
// construction through the driver entry point (no libcuda link dependency).  Included by gemm_tcgen05.cu,
// lstm_seq_tcgen05.cu and dcn_tcgen05.cu (the file names predate the Hopper port; nothing in them is tcgen05 any more).
#pragma once
#include "common.cuh"
#include <cuda.h>
#include <cuda_bf16.h>

namespace {
using namespace mr;
typedef __nv_bfloat16 bf16;

constexpr int BM = 128;
constexpr int BK = 64;             // 64 bf16 = 128 bytes = one swizzle atom
constexpr int UMMA_K = 16;           // K depth of one wgmma instruction (bf16)
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

// D[64 x N] (+)= A[64 x 16] * B[16 x N], bf16 operands through shared-memory descriptors, fp32 accumulator fragment in
// registers.  TA / TB = 1: the operand is MN-major in shared memory (the instruction's transpose bits).
template <int N> struct Wgmma;
template <> struct Wgmma<32> {
    template <int TA, int TB>
    static __device__ __forceinline__ void mma(float (&d)[16], uint64_t ad, uint64_t bd, uint32_t scale_d) {
        asm volatile(
            "{\n"
            ".reg .pred p;\n"
            "setp.ne.b32 p, %18, 0;\n"
            "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
            "%16, %17, p, 1, 1, %19, %20;\n"
            "}\n"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
            : "l"(ad), "l"(bd), "r"(scale_d), "n"(TA), "n"(TB));
    }
};
template <> struct Wgmma<64> {
    template <int TA, int TB>
    static __device__ __forceinline__ void mma(float (&d)[32], uint64_t ad, uint64_t bd, uint32_t scale_d) {
        asm volatile(
            "{\n"
            ".reg .pred p;\n"
            "setp.ne.b32 p, %34, 0;\n"
            "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
            "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
            "%32, %33, p, 1, 1, %35, %36;\n"
            "}\n"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
              "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
              "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
            : "l"(ad), "l"(bd), "r"(scale_d), "n"(TA), "n"(TB));
    }
};
template <> struct Wgmma<128> {
    template <int TA, int TB>
    static __device__ __forceinline__ void mma(float (&d)[64], uint64_t ad, uint64_t bd, uint32_t scale_d) {
        asm volatile(
            "{\n"
            ".reg .pred p;\n"
            "setp.ne.b32 p, %66, 0;\n"
            "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
            "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
            "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
            "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
            "%64, %65, p, 1, 1, %67, %68;\n"
            "}\n"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
              "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
              "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
              "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
              "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
              "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
              "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
              "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
            : "l"(ad), "l"(bd), "r"(scale_d), "n"(TA), "n"(TB));
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
    template <int TA, int TB>
    __device__ __forceinline__ void mma(uint64_t a_lo, uint64_t a_hi, uint64_t b, uint32_t accumulate) {
        Wgmma<BN>::template mma<TA, TB>(d[0], a_lo, b, accumulate);
        Wgmma<BN>::template mma<TA, TB>(d[1], a_hi, b, accumulate);
    }
    // The same step as four 64-column instructions (b_lo / b_hi: the operand's two 64-column halves), for kernels whose
    // 768 threads leave too few registers per thread for the operands of one 128-column instruction.
    template <int TA, int TB>
    __device__ __forceinline__ void mma_halves(uint64_t a_lo, uint64_t a_hi, uint64_t b_lo, uint64_t b_hi, uint32_t accumulate) {
        static_assert(BN == 128, "two 64-column halves");
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            Wgmma<64>::template mma<TA, TB>(reinterpret_cast<float (&)[32]>(d[half][0]), half ? a_hi : a_lo, b_lo, accumulate);
            Wgmma<64>::template mma<TA, TB>(reinterpret_cast<float (&)[32]>(d[half][32]), half ? a_hi : a_lo, b_hi, accumulate);
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

// MUFU.TANH: one instruction, ~2^-11 relative error -- far below bf16 resolution of the stored activations
__device__ __forceinline__ float tanh_fast(float x) { float y; asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float sigmoid_fast(float x) { return fmaf(0.5f, tanh_fast(0.5f * x), 0.5f); }


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


}  // namespace
