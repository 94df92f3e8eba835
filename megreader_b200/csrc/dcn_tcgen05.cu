// Deformable convolution v1 / v2 FORWARD as ONE fused implicit GEMM on wgmma (round 2).
//
//   out[b, co, p] = sum_{k, c} W[co, c, k] * mask[b, k, p] * bilinear(x[b, c], pos(b, k, p))  (+ bias)
//   (modulated_deform_conv_cuda_forward, assets/ops/dcn/src/deform_conv_cuda.cpp:486-564; K8 deform_conv_cuda_kernel.cu:569-632)
//
// The unfused path (csrc/dcn.cu) writes the 9x column matrix to HBM and multiplies it with an fp32 GEMM.  Here the column
// matrix never exists:
//
//   GEMM view      M = output pixels (128-row tiles inside a sample), N = Cout, K = taps x channels, K index = (cb * taps + k) * 64 + cl
//                  (a 64-wide K block is ONE tap and 64 consecutive channels; the nine taps of a channel block are consecutive K
//                  blocks, so their overlapping sampling positions are served by L1).
//   A operand      produced on the fly: 512 producer threads (8 lanes per pixel row, 2 rows each) read the four corners from an NHWC copy
//                  of the input: a warp-wide float4 gather is 4 x 128 contiguous bytes; 16 gathers per thread are in flight, blend, fold the
//                  modulation mask in, and store bf16 into the 128-byte-swizzled K-major tile that wgmma.mma_async reads.
//   precision      fp32 parity (1e-4, against the reference's own kernels) with tensor cores: every value is split
//                  v = hi + lo (two bf16), and D += Ah Wh + Ah Wl + Al Wh -- three bf16 MMAs per K block, error ~2^-17 relative
//                  (the dropped Al Wl term), fp32 accumulation in the MMA warpgroup's registers.
//   B operand      weights re-packed per call to [Cout][k * C + c] bf16 (hi and lo), tiles by 2-D TMA.
//   epilogue       accumulator tile (shared memory) -> registers -> NCHW output: a warp's 32 lanes are 32 consecutive pixels of one output channel, so
//                  every store instruction is one coalesced 128-byte row; bias added on the way.
//
// Requirements of this path: group = 1, deformable_group = 1, C % 64 == 0, Cout % 128 == 0 (the ResNet-50 DCN units of
// backbones/resnet.py:136-165 are C = Cout = 128 / 256 / 512); anything else uses the round-1 kernels in dcn.cu.
// The offset / mask indexing quirk (flat (Ho,Wo) strides inside a possibly larger per-sample slab, SURVEY.md App. B2.1) is kept.
#include "wgmma.cuh"
#include <math.h>
#include <stdlib.h>
#include <algorithm>

namespace {

struct DcnFArgs {
    const float *xh;          // [B][H][W][C] fp32
    const float *off, *msk;   // reference layout, per-sample slabs
    const float *bias;
    float *out;               // [B][Cout][Ho*Wo]
    int64_t off_bs, mask_bs;
    int B, C, H, W, Cout, kh, kw, sh, sw, ph, pw, dh, dw, Ho, Wo, P;
    int tiles_per_sample, tiles_x, ncb, nkb;     // 8 x 16 pixel tiles; ncb = C / 64 channel blocks, nkb = kh*kw*ncb K blocks
};

template <int BN, int STAGES>
struct DcnSmem {
    static constexpr int A_BYTES = BM * BK * 2;               // one of (hi, lo)
    static constexpr int B_BYTES = BN * BK * 2;
    static constexpr int STAGE_BYTES = 2 * A_BYTES + 2 * B_BYTES;
    static constexpr int BAR_OFF = STAGES * STAGE_BYTES;
    static constexpr int TAP_OFF = BAR_OFF + 128;             // barriers live in the first 128 bytes
    static constexpr int total(int taps) { return TAP_OFF + BM * taps * 24 + 1024; }   // + tap table (16 + 8 bytes / entry)
};

constexpr int kProducerThreads = 512;      // 16 warps x (4 rows x 8 channel lanes) x 2 row quads = 128 rows
constexpr int kDcnMma0 = 640;                 // producer warps end at 576; padded to a warpgroup boundary
constexpr int kDcnThreads = kDcnMma0 + kMmaThreads;

__device__ __forceinline__ void mbar_arrive_cta(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

template <int BN, int STAGES>
__global__ void __launch_bounds__(kDcnThreads, 1)
dcn_fwd_tcgen05_kernel(const __grid_constant__ CUtensorMap tmWh, const __grid_constant__ CUtensorMap tmWl, DcnFArgs a) {
    using L = DcnSmem<BN, STAGES>;
    extern __shared__ unsigned char smem_raw[];
    unsigned char *smem = (unsigned char *)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint64_t *full = (uint64_t *)(smem + L::BAR_OFF);
    uint64_t *empty = full + STAGES;
    uint64_t *tmem_full = empty + STAGES;
    float4 *tapw = (float4 *)(smem + L::TAP_OFF);             // [taps][128] bilinear weights
    uint2 *tapc = (uint2 *)(tapw + BM * a.kh * a.kw);         // [taps][128] clamped corner rows / columns
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int b = blockIdx.x / a.tiles_per_sample;
    const int tile = blockIdx.x - b * a.tiles_per_sample;
    // a tile is 8 rows x 16 columns of output pixels (tile row r = (r >> 4, r & 15)): the sampling footprint of a compact
    // block is ~half that of a 2 x 64 strip, which matters because the gathers live in what is left of L1 next to 200 KB of smem
    const int ty0 = (tile / a.tiles_x) * 8, tx0 = (tile % a.tiles_x) * 16;
    const int n0 = blockIdx.y * BN;
    const int nkb = a.nkb;

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&tmWh);
        tma_prefetch_desc(&tmWl);
        for (int s = 0; s < STAGES; ++s) { mbar_init(full + s, 1 + kProducerThreads); mbar_init(empty + s, 1); }
        mbar_init(tmem_full, 1);
        fence_barrier_init();
    }
    __syncthreads();
    float *acc_tile = (float *)smem;                         // laid over the drained operand ring when the K loop is over

    // 768 threads leave 80 registers each: the MMA warpgroup takes what its 128 accumulator registers need from the others
    if (threadIdx.x >= kDcnMma0) {
        reg_inc<160>();
        // ------------------------------------------------------------ MMA warpgroup: D += Ah Wh + Ah Wl + Al Wh
        static_assert(BN == 128, "one warpgroup holds a 128 x 128 accumulator");
        const int mt = threadIdx.x - kDcnMma0;
        AccTile<BN> acc;
        uint64_t *pending = nullptr;
        for (int i = 0; i < nkb; ++i) {
            const int s = i % STAGES;
            mbar_wait(full + s, (i / STAGES) & 1);
            const uint32_t ah = smem_u32(smem + s * L::STAGE_BYTES);
            const uint32_t al = ah + L::A_BYTES;
            const uint32_t bh = al + L::A_BYTES;
            const uint32_t bl = bh + L::B_BYTES;
            wgmma_fence();
#pragma unroll
            for (int pass = 0; pass < 3; ++pass) {
                const uint32_t aa = pass == 2 ? al : ah, bb = pass == 1 ? bl : bh;
#pragma unroll
                for (int k = 0; k < BK / UMMA_K; ++k)
                    acc.template mma_halves<0, 0>(make_desc(aa + k * 32, 16, 1024), make_desc(aa + 64 * 128 + k * 32, 16, 1024),
                                                  make_desc(bb + k * 32, 16, 1024), make_desc(bb + 64 * 128 + k * 32, 16, 1024),
                                                  (i | pass | k) != 0);
            }
            wgmma_commit();
            wgmma_wait<1>();
            if (pending && mt == 0) mbar_arrive_cta(pending);
            pending = empty + s;
        }
        wgmma_wait<0>();
        if (pending && mt == 0) mbar_arrive_cta(pending);
        mma_group_sync();
        acc.store(acc_tile, mt);
        mma_group_sync();
        if (mt == 0) mbar_arrive_cta(tmem_full);
        return;
    }
    reg_dec<64>();
    if (warp == 0) {
        // ------------------------------------------------------------ weight tiles (hi and lo) by TMA
        if (elect_one()) {
            for (int i = 0; i < nkb; ++i) {
                const int s = i % STAGES;
                mbar_wait(empty + s, ((i / STAGES) & 1) ^ 1);
                unsigned char *st = smem + s * L::STAGE_BYTES + 2 * L::A_BYTES;
                mbar_expect_tx(full + s, 2 * L::B_BYTES);
                tma_load_2d(&tmWh, full + s, st, i * BK, n0);
                tma_load_2d(&tmWl, full + s, st + L::B_BYTES, i * BK, n0);
            }
        }
    } else if (warp >= 2 && threadIdx.x < 64 + kProducerThreads) {
        // ------------------------------------------------------------ producers: bilinear gather -> swizzled bf16 tiles
        // Thread mapping: 8 lanes share a pixel row and split its 64 channels (lane j: channels 4j..4j+3 and 32+4j..32+4j+3),
        // 4 rows per warp instruction, 2 such row quads per warp.  A warp-wide float4 gather therefore touches 4 x 128
        // contiguous bytes (4 L1 wavefronts); with lanes = 32 different pixels it was 32 separate half-used sectors and
        // the gathers were bound by the L1 data stage.
        const int pwp = warp - 2;                             // producer warp 0..15
        const int sub = lane >> 3, j = lane & 7;
        struct Row { const float4 *q1, *q2, *q3, *q4; float w1, w2, w3, w4; };
        const float *xb = a.xh + (int64_t)b * a.H * a.W * a.C + j * 4;
        // ---- tap table: the bilinear set-up of every (row, tap) of this tile is computed ONCE (one entry per producer thread
        // and pass) instead of by each of the 8 lanes that share a row: 4 weights (mask and validity folded in) + 4 clamped
        // corner coordinates (uint16), 24 bytes per entry.
        {
            const int nent = BM * a.kh * a.kw;
            const float *offb = a.off + (int64_t)b * a.off_bs;
            const float *mskb = a.msk ? a.msk + (int64_t)b * a.mask_bs : nullptr;
            for (int e = threadIdx.x - 64; e < nent; e += kProducerThreads) {
                const int k = e / BM, r = e - k * BM;
                const int py = ty0 + (r >> 4), px = tx0 + (r & 15);
                const bool rok = py < a.Ho && px < a.Wo;
                const int ho = rok ? py : a.Ho - 1, wo = rok ? px : a.Wo - 1;
                const int pc = ho * a.Wo + wo;
                const int ti = k / a.kw, tj = k - ti * a.kw;
                const float oh = __ldg(offb + (int64_t)(2 * k) * a.P + pc);
                const float ow = __ldg(offb + (int64_t)(2 * k + 1) * a.P + pc);
                const float m = mskb ? __ldg(mskb + (int64_t)k * a.P + pc) : 1.f;
                const float hy = (float)(ho * a.sh - a.ph + ti * a.dh) + oh;
                const float wx = (float)(wo * a.sw - a.pw + tj * a.dw) + ow;
                // dmcn_im2col_bilinear (deform_conv_cuda_kernel.cu:466-496): zero outside (-1,H) x (-1,W), corners outside dropped
                const bool inside = rok && hy > -1.f && wx > -1.f && hy < (float)a.H && wx < (float)a.W;
                const int hl = (int)floorf(hy), wl = (int)floorf(wx);
                const int hh = hl + 1, wh = wl + 1;
                const float lh = hy - hl, lw = wx - wl, uh = 1.f - lh, uw = 1.f - lw;
                const bool m1 = inside && hl >= 0 && wl >= 0, m2 = inside && hl >= 0 && wh <= a.W - 1;
                const bool m3 = inside && hh <= a.H - 1 && wl >= 0, m4 = inside && hh <= a.H - 1 && wh <= a.W - 1;
                tapw[e] = make_float4(m1 ? uh * uw * m : 0.f, m2 ? uh * lw * m : 0.f, m3 ? lh * uw * m : 0.f, m4 ? lh * lw * m : 0.f);
                const int y0 = min(max(hl, 0), a.H - 1), y1 = min(max(hh, 0), a.H - 1);
                const int x0 = min(max(wl, 0), a.W - 1), x1 = min(max(wh, 0), a.W - 1);
                tapc[e] = make_uint2((unsigned)y0 | ((unsigned)y1 << 16), (unsigned)x0 | ((unsigned)x1 << 16));
            }
            asm volatile("bar.sync 1, %0;" ::"n"(kProducerThreads) : "memory");      // producers only
        }
        int rrow[2];
#pragma unroll
        for (int u = 0; u < 2; ++u) rrow[u] = pwp * 8 + u * 4 + sub;
        int kb = 0;
        // K order: channel block outermost, tap inside -- consecutive K blocks gather the SAME 64 channels at the nine taps'
        // overlapping positions, so the lines stay in L1 across taps
        for (int cc = 0; cc < a.ncb; ++cc)
        for (int k = 0; k < a.kh * a.kw; ++k, ++kb) {
            Row rw[2];
#pragma unroll
            for (int u = 0; u < 2; ++u) {
                const float4 wv = tapw[k * BM + rrow[u]];
                const uint2 cv = tapc[k * BM + rrow[u]];
                rw[u].w1 = wv.x; rw[u].w2 = wv.y; rw[u].w3 = wv.z; rw[u].w4 = wv.w;
                const int y0 = (int)(cv.x & 0xffffu) * a.W, y1 = (int)(cv.x >> 16) * a.W;
                const int x0 = (int)(cv.y & 0xffffu), x1 = (int)(cv.y >> 16);
                rw[u].q1 = reinterpret_cast<const float4 *>(xb + (int64_t)(y0 + x0) * a.C);
                rw[u].q2 = reinterpret_cast<const float4 *>(xb + (int64_t)(y0 + x1) * a.C);
                rw[u].q3 = reinterpret_cast<const float4 *>(xb + (int64_t)(y1 + x0) * a.C);
                rw[u].q4 = reinterpret_cast<const float4 *>(xb + (int64_t)(y1 + x1) * a.C);
            }
            {
                // all 16 gathers of this thread are issued before the slot wait and before any use
                float4 x1[2][2], x2[2][2], x3[2][2], x4[2][2];
                const int c4 = cc * (BK / 4);
#pragma unroll
                for (int u = 0; u < 2; ++u)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        x1[u][e] = __ldg(rw[u].q1 + c4 + e * 8); x2[u][e] = __ldg(rw[u].q2 + c4 + e * 8);
                        x3[u][e] = __ldg(rw[u].q3 + c4 + e * 8); x4[u][e] = __ldg(rw[u].q4 + c4 + e * 8);
                    }
                const int s = kb % STAGES;
                mbar_wait(empty + s, ((kb / STAGES) & 1) ^ 1);
                const uint32_t ah_s = smem_u32(smem + s * L::STAGE_BYTES);
#pragma unroll
                for (int u = 0; u < 2; ++u) {
                    const uint32_t row_off = (uint32_t)rrow[u] * 128u, sw = (uint32_t)(rrow[u] & 7);
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const float v0 = rw[u].w1 * x1[u][e].x + rw[u].w2 * x2[u][e].x + rw[u].w3 * x3[u][e].x + rw[u].w4 * x4[u][e].x;
                        const float v1 = rw[u].w1 * x1[u][e].y + rw[u].w2 * x2[u][e].y + rw[u].w3 * x3[u][e].y + rw[u].w4 * x4[u][e].y;
                        const float v2 = rw[u].w1 * x1[u][e].z + rw[u].w2 * x2[u][e].z + rw[u].w3 * x3[u][e].z + rw[u].w4 * x4[u][e].z;
                        const float v3 = rw[u].w1 * x1[u][e].w + rw[u].w2 * x2[u][e].w + rw[u].w3 * x3[u][e].w + rw[u].w4 * x4[u][e].w;
                        uint2 hi, lo;
                        __nv_bfloat162 *h2 = reinterpret_cast<__nv_bfloat162 *>(&hi);
                        __nv_bfloat162 *l2 = reinterpret_cast<__nv_bfloat162 *>(&lo);
                        h2[0] = __floats2bfloat162_rn(v0, v1);
                        h2[1] = __floats2bfloat162_rn(v2, v3);
                        const float2 f0 = __bfloat1622float2(h2[0]), f1 = __bfloat1622float2(h2[1]);
                        l2[0] = __floats2bfloat162_rn(v0 - f0.x, v1 - f0.y);
                        l2[1] = __floats2bfloat162_rn(v2 - f1.x, v3 - f1.y);
                        // channels e*32 + 4j .. +3 -> 16-byte chunk e*4 + j/2 of the row (swizzled), 8-byte half j & 1
                        const uint32_t o = row_off + ((((uint32_t)(e * 4 + (j >> 1))) ^ sw) << 4) + (uint32_t)(j & 1) * 8u;
                        asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(ah_s + o), "r"(hi.x), "r"(hi.y) : "memory");
                        asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(ah_s + (uint32_t)L::A_BYTES + o), "r"(lo.x), "r"(lo.y) : "memory");
                    }
                }
                fence_proxy_async();                          // generic-proxy smem writes -> visible to wgmma
                mbar_arrive_cta(full + s);
            }
        }
        // ------------------------------------------------------------ epilogue: accumulator tile -> NCHW (+ bias); 4 warps per 32-row quarter
        const int q = warp & 3;                               // 32-row quarter of the tile this warp stores
        const int part = (warp - 2) >> 2;                     // which quarter of the BN columns (4 warps share a row quarter)
        const int er = q * 32 + lane;
        const int ey = ty0 + (er >> 4), ex = tx0 + (er & 15);
        const int prow = (ey < a.Ho && ex < a.Wo) ? ey * a.Wo + ex : a.P;
        mbar_wait(tmem_full, 0);
        float *ob = a.out + ((int64_t)b * a.Cout + n0) * a.P + prow;
#pragma unroll 1
        for (int c = part * (BN / 128); c < (part + 1) * (BN / 128); ++c) {
            uint32_t rr[32];
            acc_ld<32>(acc_tile, AccTile<BN>::LD, q * 32, c * 32, rr);
            if (prow < a.P) {
#pragma unroll
                for (int j = 0; j < 32; ++j) {
                    const int co = c * 32 + j;
                    float v = __uint_as_float(rr[j]);
                    if (a.bias) v += __ldg(a.bias + n0 + co);
                    ob[(int64_t)co * a.P] = v;
                }
            }
        }
    }
}

// =====================================================================================================
// Fused WEIGHT GRADIENT (round 2):  gw[co, c, k] += scale * sum_{b,p} go[b, co, p] * col[b, p, (c, k)]
//   (deform_conv_cuda.cpp:645-658 / :373-484: im2col of every sample + one SGEMM per sample in the reference)
// The column matrix is produced exactly as in the forward (same producer threads, same swizzled tile [128 pixels][64 (tap, channels)])
// but now it is the MN-major B operand of  D[co (128), kc (64)] += go^T[co, p] * col[p, kc]  with the PIXELS as the reduction
// dimension.  One CTA owns one 64-wide (tap, channel block) slice and one 128-channel slice of Cout and walks over a strided subset
// of the pixel tiles (split-K); the A operand is grad_output re-tiled to [b * tiles + tile][co][128 pixels in tile order] and split
// into bf16 hi / lo by a small pre-pass, so that one pixel tile of it is a plain 2-D TMA box.  fp32 atomics at the end.
// =====================================================================================================
struct DcnWArgs {
    const float *xh, *off, *msk;
    float *gw;                // [Cout][C][kh*kw] fp32, accumulated
    int64_t off_bs, mask_bs;
    float scale;
    int B, C, H, W, Cout, kh, kw, sh, sw, ph, pw, dh, dw, Ho, Wo, P;
    int tiles_per_sample, tiles_x, ncb, nkb, ntiles, splits;
};

struct DcnWSmem {
    static constexpr int B_BYTES = BM * BK * 2;               // produced tile, one of (hi, lo): [128 pixels][64 kc]
    static constexpr int A_BYTES = BM * BM * 2;               // go tile, one of (hi, lo): [128 co][128 pixels] = two 64-pixel atoms
    static constexpr int STAGES = 2;                          // of the produced operand; the TMA operand has ONE buffer: its load for tile
    static constexpr int A_OFF = STAGES * 2 * B_BYTES;        // i + 1 is issued when the MMAs of tile i retire and lands while tile i + 1
    static constexpr int BAR_OFF = A_OFF + 2 * A_BYTES;       // is being gathered -- 64 KB less shared memory = 64 KB more L1 for the gathers
    static constexpr int TAP_OFF = BAR_OFF + 128;
    static constexpr int TOTAL = TAP_OFF + 2 * BM * 24 + 1024;   // one tap-table row set per tile parity
};

__global__ void __launch_bounds__(kDcnThreads, 1)
dcn_wgrad_tcgen05_kernel(const __grid_constant__ CUtensorMap tmGh, const __grid_constant__ CUtensorMap tmGl, DcnWArgs a) {
    using L = DcnWSmem;
    constexpr int STAGES = L::STAGES;
    extern __shared__ unsigned char smem_raw[];
    unsigned char *smem = (unsigned char *)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint64_t *full = (uint64_t *)(smem + L::BAR_OFF);         // produced operand: full (512 producer arrivals) / empty (MMA commit)
    uint64_t *empty = full + STAGES;
    uint64_t *a_full = empty + STAGES, *a_empty = a_full + 1;  // TMA operand, single buffer
    uint64_t *tmem_full = a_empty + 1;
    float4 *tapw_all = (float4 *)(smem + L::TAP_OFF);         // [STAGES][128]
    uint2 *tapc_all = (uint2 *)(tapw_all + STAGES * BM);      // [STAGES][128]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int kb = blockIdx.x;                                // K block of the forward GEMM: (channel block, tap)
    const int cc = kb / (a.kh * a.kw), k = kb - cc * (a.kh * a.kw);
    const int co0 = blockIdx.z * BM;
    const int nt = (a.ntiles - (int)blockIdx.y + a.splits - 1) / a.splits;      // pixel tiles of this CTA: y, y + splits, ...
    constexpr int BN = 64;

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&tmGh);
        tma_prefetch_desc(&tmGl);
        for (int s = 0; s < STAGES; ++s) { mbar_init(full + s, kProducerThreads); mbar_init(empty + s, 1); }
        mbar_init(a_full, 1); mbar_init(a_empty, 1);
        mbar_init(tmem_full, 1);
        fence_barrier_init();
    }
    __syncthreads();
    float *acc_tile = (float *)smem;                         // laid over the drained operand ring when the loop is over

    if (warp == 0) {
        if (elect_one()) {
            for (int i = 0; i < nt; ++i) {
                const int gt = (int)blockIdx.y + i * a.splits;
                mbar_wait(a_empty, (i & 1) ^ 1);
                unsigned char *st = smem + L::A_OFF;
                mbar_expect_tx(a_full, 2 * L::A_BYTES);
                const int row = gt * a.Cout + co0;                        // rows of the re-tiled grad_output: (tile, co)
                tma_load_2d(&tmGh, a_full, st, 0, row);
                tma_load_2d(&tmGh, a_full, st + BM * 128, 64, row);
                tma_load_2d(&tmGl, a_full, st + L::A_BYTES, 0, row);
                tma_load_2d(&tmGl, a_full, st + L::A_BYTES + BM * 128, 64, row);
            }
        }
    } else if (threadIdx.x >= kDcnMma0) {
        // A K-major (pixels contiguous), B MN-major (kc contiguous)
        const int mt = threadIdx.x - kDcnMma0;
        AccTile<BN> acc;
        for (int i = 0; i < nt; ++i) {
            const int s = i % STAGES;
            mbar_wait(full + s, (i / STAGES) & 1);
            mbar_wait(a_full, i & 1);
            const uint32_t bh = smem_u32(smem + s * 2 * L::B_BYTES);
            const uint32_t bl = bh + L::B_BYTES;
            const uint32_t ah = smem_u32(smem + L::A_OFF);
            const uint32_t al = ah + L::A_BYTES;
            wgmma_fence();
#pragma unroll
            for (int pass = 0; pass < 3; ++pass) {
                const uint32_t aa = pass == 2 ? al : ah, bb = pass == 1 ? bl : bh;       // Ah Bh, Ah Bl, Al Bh
#pragma unroll
                for (int j = 0; j < BM / UMMA_K; ++j) {                                   // 8 steps of 16 pixels
                    const uint32_t ak = aa + (j >> 2) * (BM * 128) + (j & 3) * 32;
                    acc.mma<0, 1>(make_desc(ak, 16, 1024), make_desc(ak + 64 * 128, 16, 1024), make_desc(bb + j * 2048, BM * 128, 1024),
                                  (i | pass | j) != 0);
                }
            }
            wgmma_commit();
            wgmma_wait<0>();
            if (mt == 0) { mbar_arrive_cta(empty + s); mbar_arrive_cta(a_empty); }
        }
        if (nt > 0) {
            mma_group_sync();
            acc.store(acc_tile, mt);
            mma_group_sync();
            if (mt == 0) mbar_arrive_cta(tmem_full);
        }
    } else if (warp >= 2 && threadIdx.x < 64 + kProducerThreads) {
        const int pwp = warp - 2;
        const int sub = lane >> 3, j = lane & 7;
        const int ptid = threadIdx.x - 64;
        int rrow[2];
#pragma unroll
        for (int u = 0; u < 2; ++u) rrow[u] = pwp * 8 + u * 4 + sub;
        const int ti = k / a.kw, tj = k - ti * a.kw;
        // tap table of one pixel tile (128 rows, this CTA's tap): raw offset / mask loads and the derived weights / corners are split so
        // that the loads of tile i + 1 are in flight while tile i is gathered
        auto tap_load = [&](int gt, float &oh, float &ow, float &m) {
            const int bb = gt / a.tiles_per_sample, tile = gt - bb * a.tiles_per_sample;
            const int r = ptid;
            const int py = (tile / a.tiles_x) * 8 + (r >> 4), px = (tile % a.tiles_x) * 16 + (r & 15);
            const bool rok = py < a.Ho && px < a.Wo;
            const int pc = (rok ? py : a.Ho - 1) * a.Wo + (rok ? px : a.Wo - 1);
            const float *offb = a.off + (int64_t)bb * a.off_bs;
            oh = __ldg(offb + (int64_t)(2 * k) * a.P + pc);
            ow = __ldg(offb + (int64_t)(2 * k + 1) * a.P + pc);
            m = a.msk ? __ldg(a.msk + (int64_t)bb * a.mask_bs + (int64_t)k * a.P + pc) : 1.f;
        };
        auto tap_store = [&](int gt, int slot, float oh, float ow, float m) {
            const int bb = gt / a.tiles_per_sample, tile = gt - bb * a.tiles_per_sample;
            const int r = ptid;
            const int py = (tile / a.tiles_x) * 8 + (r >> 4), px = (tile % a.tiles_x) * 16 + (r & 15);
            const bool rok = py < a.Ho && px < a.Wo;
            const int ho = rok ? py : a.Ho - 1, wo = rok ? px : a.Wo - 1;
            const float hy = (float)(ho * a.sh - a.ph + ti * a.dh) + oh;
            const float wx = (float)(wo * a.sw - a.pw + tj * a.dw) + ow;
            const bool inside = rok && hy > -1.f && wx > -1.f && hy < (float)a.H && wx < (float)a.W;
            const int hl = (int)floorf(hy), wl = (int)floorf(wx);
            const int hh = hl + 1, wh = wl + 1;
            const float lh = hy - hl, lw = wx - wl, uh = 1.f - lh, uw = 1.f - lw;
            const bool m1 = inside && hl >= 0 && wl >= 0, m2 = inside && hl >= 0 && wh <= a.W - 1;
            const bool m3 = inside && hh <= a.H - 1 && wl >= 0, m4 = inside && hh <= a.H - 1 && wh <= a.W - 1;
            tapw_all[slot * BM + r] = make_float4(m1 ? uh * uw * m : 0.f, m2 ? uh * lw * m : 0.f, m3 ? lh * uw * m : 0.f, m4 ? lh * lw * m : 0.f);
            const int y0 = min(max(hl, 0), a.H - 1), y1 = min(max(hh, 0), a.H - 1);
            const int x0 = min(max(wl, 0), a.W - 1), x1 = min(max(wh, 0), a.W - 1);
            tapc_all[slot * BM + r] = make_uint2((unsigned)y0 | ((unsigned)y1 << 16), (unsigned)x0 | ((unsigned)x1 << 16));
        };
        if (ptid < BM && nt > 0) {
            float oh, ow, m;
            tap_load((int)blockIdx.y, oh, ow, m);
            tap_store((int)blockIdx.y, 0, oh, ow, m);
        }
        asm volatile("bar.sync 1, %0;" ::"n"(kProducerThreads) : "memory");
        for (int i = 0; i < nt; ++i) {
            const int s = i % STAGES;
            const int gt = (int)blockIdx.y + i * a.splits;
            const int b = gt / a.tiles_per_sample;
            const float4 *tapw = tapw_all + (i & 1) * BM;
            const uint2 *tapc = tapc_all + (i & 1) * BM;
            const bool prep = ptid < BM && i + 1 < nt;
            float noh = 0.f, now = 0.f, nm = 0.f;
            if (prep) tap_load(gt + a.splits, noh, now, nm);
            mbar_wait(empty + s, ((i / STAGES) & 1) ^ 1);
            const float *xb = a.xh + (int64_t)b * a.H * a.W * a.C + j * 4;
            const int c4 = cc * (BK / 4);
            float4 x1[2][2], x2[2][2], x3[2][2], x4[2][2];
            float4 wv[2];
#pragma unroll
            for (int u = 0; u < 2; ++u) {
                wv[u] = tapw[rrow[u]];
                const uint2 cv = tapc[rrow[u]];
                const int y0 = (int)(cv.x & 0xffffu) * a.W, y1 = (int)(cv.x >> 16) * a.W;
                const int x0 = (int)(cv.y & 0xffffu), xx1 = (int)(cv.y >> 16);
                const float4 *q1 = reinterpret_cast<const float4 *>(xb + (int64_t)(y0 + x0) * a.C);
                const float4 *q2 = reinterpret_cast<const float4 *>(xb + (int64_t)(y0 + xx1) * a.C);
                const float4 *q3 = reinterpret_cast<const float4 *>(xb + (int64_t)(y1 + x0) * a.C);
                const float4 *q4 = reinterpret_cast<const float4 *>(xb + (int64_t)(y1 + xx1) * a.C);
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    x1[u][e] = __ldg(q1 + c4 + e * 8); x2[u][e] = __ldg(q2 + c4 + e * 8);
                    x3[u][e] = __ldg(q3 + c4 + e * 8); x4[u][e] = __ldg(q4 + c4 + e * 8);
                }
            }
            const uint32_t bh_s = smem_u32(smem + s * 2 * L::B_BYTES);
#pragma unroll
            for (int u = 0; u < 2; ++u) {
                const uint32_t row_off = (uint32_t)rrow[u] * 128u, sw = (uint32_t)(rrow[u] & 7);
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const float v0 = wv[u].x * x1[u][e].x + wv[u].y * x2[u][e].x + wv[u].z * x3[u][e].x + wv[u].w * x4[u][e].x;
                    const float v1 = wv[u].x * x1[u][e].y + wv[u].y * x2[u][e].y + wv[u].z * x3[u][e].y + wv[u].w * x4[u][e].y;
                    const float v2 = wv[u].x * x1[u][e].z + wv[u].y * x2[u][e].z + wv[u].z * x3[u][e].z + wv[u].w * x4[u][e].z;
                    const float v3 = wv[u].x * x1[u][e].w + wv[u].y * x2[u][e].w + wv[u].z * x3[u][e].w + wv[u].w * x4[u][e].w;
                    uint2 hi, lo;
                    __nv_bfloat162 *h2 = reinterpret_cast<__nv_bfloat162 *>(&hi);
                    __nv_bfloat162 *l2 = reinterpret_cast<__nv_bfloat162 *>(&lo);
                    h2[0] = __floats2bfloat162_rn(v0, v1);
                    h2[1] = __floats2bfloat162_rn(v2, v3);
                    const float2 f0 = __bfloat1622float2(h2[0]), f1 = __bfloat1622float2(h2[1]);
                    l2[0] = __floats2bfloat162_rn(v0 - f0.x, v1 - f0.y);
                    l2[1] = __floats2bfloat162_rn(v2 - f1.x, v3 - f1.y);
                    const uint32_t o = row_off + ((((uint32_t)(e * 4 + (j >> 1))) ^ sw) << 4) + (uint32_t)(j & 1) * 8u;
                    asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(bh_s + o), "r"(hi.x), "r"(hi.y) : "memory");
                    asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(bh_s + (uint32_t)L::B_BYTES + o), "r"(lo.x), "r"(lo.y) : "memory");
                }
            }
            fence_proxy_async();
            mbar_arrive_cta(full + s);
            if (prep) tap_store(gt + a.splits, (i + 1) & 1, noh, now, nm);
            asm volatile("bar.sync 1, %0;" ::"n"(kProducerThreads) : "memory");
        }
        // ---- epilogue: D[co][kc] -> gw[co][c][k] (fp32 atomics; 4 warps per row quarter, 16 columns each)
        const int q = warp & 3, part = (warp - 2) >> 2;
        const int co = co0 + q * 32 + lane;
        if (nt > 0) {
            mbar_wait(tmem_full, 0);
            uint32_t rr[16];
            acc_ld<16>(acc_tile, AccTile<BN>::LD, q * 32, part * 16, rr);
            if (co < a.Cout) {
                float *gp = a.gw + ((int64_t)co * a.C + cc * BK + part * 16) * (a.kh * a.kw) + k;
#pragma unroll
                for (int e = 0; e < 16; ++e) atomicAdd(gp + (int64_t)e * (a.kh * a.kw), a.scale * __uint_as_float(rr[e]));
            }
        }
    }
}

// =====================================================================================================
// Fused DATA GRADIENT (round 2): grad_input, grad_offset, grad_mask without the column-gradient matrix
//   colg[b, p, (k, c)] = sum_co go[b, co, p] * W[co, c, k]          (deform_conv_cuda.cpp:611-614, an SGEMM per sample in the reference)
//   grad_input  += bilinear scatter of colg * mask                  (K9,  deform_conv_cuda_kernel.cu:634-692)
//   grad_offset  = sum_c colg * mask * d bilinear / d position      (K10, :694-766)
//   grad_mask    = sum_c colg * bilinear(x)                         (K10, :752)
// One CTA owns one 8 x 16 pixel tile and a subset of the taps.  For a tap and a 128-channel chunk the 128 x 128 block of colg is one
// wgmma GEMM over Cout (A = re-tiled grad_output, MN-major: pixels contiguous; B = the forward's packed weights read MN-major:
// (tap, channel) contiguous; bf16 hi / lo, three MMAs per K block) into the MMA warpgroup's register accumulator, published as a shared-memory tile.  The 16 epilogue warps move
// it through a swizzled fp32 staging tile to the forward's 8-lanes-per-pixel mapping, gather the four corners from the NHWC input
// (128 contiguous bytes per 8 lanes), form the three per-pixel sums and scatter into an NHWC fp32 copy of grad_input with 16-byte
// vector reductions (red.global.add.v4.f32), which a transpose-add folds into the caller's NCHW tensor.
// =====================================================================================================
struct DcnDArgs {
    const float *xh, *off, *msk;
    float *gxh;                // [B][H][W][C] fp32, zero-filled; nullptr = no grad_input wanted
    float *goff, *gmask;       // reference layouts (flat (Ho, Wo) strides inside per-sample slabs); either may be nullptr
    int64_t off_bs, mask_bs, goff_bs, gmask_bs;
    int B, C, H, W, Cout, kh, kw, sh, sw, ph, pw, dh, dw, Ho, Wo, P;
    int tiles_per_sample, tiles_x, nch, nkk, tap_splits;     // nch = C / 128 channel chunks, nkk = Cout / 32 K blocks
};

struct DcnDSmem {
    static constexpr int BN = 128;
    static constexpr int KB = 32;                             // output channels (the reduction dimension) per pipeline stage
    static constexpr int OP_BYTES = KB * 128 * 2;             // one operand tile, one of (hi, lo): [32 co][128 (pixels | kc)] = 8 KB
    static constexpr int STAGE_BYTES = 4 * OP_BYTES;          // A hi, A lo, B hi, B lo
    static constexpr int STAGES = 2;                          // small on purpose: the epilogue's gathers want the rest of the SM's L1
    static constexpr int STG_OFF = STAGES * STAGE_BYTES;      // fp32 staging tile [128 pixels][128 channels], 16-byte chunks XOR-swizzled
    static constexpr int STG_BYTES = BM * BN * 4;
    static constexpr int ACC_OFF = STG_OFF + STG_BYTES;       // the accumulator tile the MMA warpgroup publishes
    static constexpr int BAR_OFF = ACC_OFF + (AccTile<BN>::BYTES + 127) / 128 * 128;
    static constexpr int TAB_OFF = BAR_OFF + 128;
    static constexpr int TAB_BYTES = 2 * BM * (3 * 16 + 8 + 4);          // tap tables, double-buffered by tap parity
    static constexpr int TOTAL = TAB_OFF + TAB_BYTES + 1024;
};

__device__ __forceinline__ void red_add_v4(float *p, float a, float b, float c, float d) {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

// per-(pixel row, tap) sampling data of the data-gradient epilogue (dmcn_im2col_bilinear / dmcn_get_coordinate_weight,
// deform_conv_cuda_kernel.cu:466-567, evaluated once per row instead of once per channel)
struct DcnDTab {
    float4 *w, *h, *v;      // bilinear weights of the valid corners; mask * d/dh and mask * d/dw coefficients of the four corner values
    uint2 *c;               // clamped corner rows / columns
    float *m;               // modulation mask
};
struct DcnDRaw { float oh, ow, m; };
__device__ __forceinline__ DcnDRaw dcn_dgrad_load_row(const DcnDArgs &a, int b, int kk, int r, int ty0, int tx0) {
    const int py = ty0 + (r >> 4), px = tx0 + (r & 15);
    const bool rok = py < a.Ho && px < a.Wo;
    const int pc = (rok ? py : a.Ho - 1) * a.Wo + (rok ? px : a.Wo - 1);
    const float *offb = a.off + (int64_t)b * a.off_bs;
    DcnDRaw v;
    v.oh = __ldg(offb + (int64_t)(2 * kk) * a.P + pc);
    v.ow = __ldg(offb + (int64_t)(2 * kk + 1) * a.P + pc);
    v.m = a.msk ? __ldg(a.msk + (int64_t)b * a.mask_bs + (int64_t)kk * a.P + pc) : 1.f;
    return v;
}
__device__ __forceinline__ void dcn_dgrad_store_row(const DcnDArgs &a, const DcnDTab &t, const DcnDRaw &v, int kk, int r, int ty0, int tx0) {
    const int ti = kk / a.kw, tj = kk - ti * a.kw;
    const int py = ty0 + (r >> 4), px = tx0 + (r & 15);
    const bool rok = py < a.Ho && px < a.Wo;
    const int ho = rok ? py : a.Ho - 1, wo = rok ? px : a.Wo - 1;
    const float m = v.m;
    const float hy = (float)(ho * a.sh - a.ph + ti * a.dh) + v.oh;
    const float wx = (float)(wo * a.sw - a.pw + tj * a.dw) + v.ow;
    const bool inside = rok && hy > -1.f && wx > -1.f && hy < (float)a.H && wx < (float)a.W;
    const int hl = (int)floorf(hy), wl = (int)floorf(wx);
    const int hh = hl + 1, wh = wl + 1;
    const float lh = hy - hl, lw = wx - wl, uh = 1.f - lh, uw = 1.f - lw;
    const float f1 = (inside && hl >= 0 && wl >= 0) ? 1.f : 0.f, f2 = (inside && hl >= 0 && wh <= a.W - 1) ? 1.f : 0.f;
    const float f3 = (inside && hh <= a.H - 1 && wl >= 0) ? 1.f : 0.f, f4 = (inside && hh <= a.H - 1 && wh <= a.W - 1) ? 1.f : 0.f;
    t.w[r] = make_float4(f1 * uh * uw, f2 * uh * lw, f3 * lh * uw, f4 * lh * lw);
    t.h[r] = make_float4(-m * uw * f1, -m * lw * f2, m * uw * f3, m * lw * f4);
    t.v[r] = make_float4(-m * uh * f1, m * uh * f2, -m * lh * f3, m * lh * f4);
    const int y0 = min(max(hl, 0), a.H - 1), y1 = min(max(hh, 0), a.H - 1);
    const int x0 = min(max(wl, 0), a.W - 1), x1 = min(max(wh, 0), a.W - 1);
    t.c[r] = make_uint2((unsigned)y0 | ((unsigned)y1 << 16), (unsigned)x0 | ((unsigned)x1 << 16));
    t.m[r] = m;
}

__global__ void __launch_bounds__(kDcnThreads, 1)
dcn_dgrad_tcgen05_kernel(const __grid_constant__ CUtensorMap tmGh, const __grid_constant__ CUtensorMap tmGl,
                         const __grid_constant__ CUtensorMap tmWh, const __grid_constant__ CUtensorMap tmWl, DcnDArgs a) {
    using L = DcnDSmem;
    constexpr int STAGES = L::STAGES;
    constexpr int BN = L::BN;
    extern __shared__ unsigned char smem_raw[];
    unsigned char *smem = (unsigned char *)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint64_t *full = (uint64_t *)(smem + L::BAR_OFF);
    uint64_t *empty = full + STAGES;
    uint64_t *acc_full = empty + STAGES;
    uint64_t *acc_empty = acc_full + 2;
    auto tab_of = [&](int tb) {
        DcnDTab t;
        unsigned char *base = smem + L::TAB_OFF + tb * (L::TAB_BYTES / 2);
        t.w = (float4 *)base; t.h = t.w + BM; t.v = t.h + BM;
        t.c = (uint2 *)(t.v + BM); t.m = (float *)(t.c + BM);
        return t;
    };
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int gt = blockIdx.x;
    const int b = gt / a.tiles_per_sample;
    const int tile = gt - b * a.tiles_per_sample;
    const int ty0 = (tile / a.tiles_x) * 8, tx0 = (tile % a.tiles_x) * 16;
    const int K = a.kh * a.kw;

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&tmGh); tma_prefetch_desc(&tmGl); tma_prefetch_desc(&tmWh); tma_prefetch_desc(&tmWl);
        for (int s = 0; s < STAGES; ++s) { mbar_init(full + s, 1); mbar_init(empty + s, 1); }
        for (int s = 0; s < 2; ++s) { mbar_init(acc_full + s, 1); mbar_init(acc_empty + s, kProducerThreads / 32); }
        fence_barrier_init();
    }
    __syncthreads();
    float *acc_tile = (float *)(smem + L::ACC_OFF);

    // 768 threads leave 80 registers each: the MMA warpgroup takes what its 128 accumulator registers need from the others
    if (threadIdx.x >= kDcnMma0) {
        reg_inc<160>();
        // both operands MN-major.  The accumulator of block n lives in registers, so its MMAs overlap the epilogue of block
        // n - 1; only the publication into the single shared tile waits until the epilogue warps have drained that block.
        const int mt = threadIdx.x - kDcnMma0;
        AccTile<BN> acc;
        int i = 0, n = 0;
        for (int kk = blockIdx.y; kk < K; kk += a.tap_splits)
            for (int h = 0; h < a.nch; ++h, ++n) {
                const int buf = n & 1;
                uint64_t *pending = nullptr;
                for (int kb = 0; kb < a.nkk; ++kb, ++i) {
                    const int s = i % STAGES;
                    mbar_wait(full + s, (i / STAGES) & 1);
                    const uint32_t ah = smem_u32(smem + s * L::STAGE_BYTES);
                    const uint32_t al = ah + L::OP_BYTES, bh = ah + 2 * L::OP_BYTES, bl = ah + 3 * L::OP_BYTES;
                    wgmma_fence();
#pragma unroll
                    for (int pass = 0; pass < 3; ++pass) {
                        const uint32_t aa = pass == 2 ? al : ah, bb = pass == 1 ? bl : bh;
#pragma unroll
                        for (int k4 = 0; k4 < L::KB / UMMA_K; ++k4)
                            acc.mma_halves<1, 1>(make_desc(aa + k4 * 2048, L::KB * 128, 1024), make_desc(aa + L::KB * 128 + k4 * 2048, L::KB * 128, 1024),
                                                 make_desc(bb + k4 * 2048, L::KB * 128, 1024), make_desc(bb + L::KB * 128 + k4 * 2048, L::KB * 128, 1024),
                                                 (kb | pass | k4) != 0);
                    }
                    wgmma_commit();
                    wgmma_wait<1>();
                    if (pending && mt == 0) mbar_arrive_cta(pending);
                    pending = empty + s;
                }
                wgmma_wait<0>();
                if (pending && mt == 0) mbar_arrive_cta(pending);
                if (n > 0) mbar_wait(acc_empty + (buf ^ 1), ((n - 1) >> 1) & 1);
                acc.store(acc_tile, mt);
                mma_group_sync();
                if (mt == 0) mbar_arrive_cta(acc_full + buf);
            }
        return;
    }
    reg_dec<64>();
    if (warp == 0) {
        if (elect_one()) {
            int i = 0;
            for (int kk = blockIdx.y; kk < K; kk += a.tap_splits)
                for (int h = 0; h < a.nch; ++h)
                    for (int kb = 0; kb < a.nkk; ++kb, ++i) {
                        const int s = i % STAGES;
                        mbar_wait(empty + s, ((i / STAGES) & 1) ^ 1);
                        unsigned char *st = smem + s * L::STAGE_BYTES;
                        mbar_expect_tx(full + s, L::STAGE_BYTES);
                        const int grow = gt * a.Cout + kb * L::KB;                         // (tile, co) rows of the re-tiled grad_output
                        tma_load_2d(&tmGh, full + s, st, 0, grow);
                        tma_load_2d(&tmGh, full + s, st + L::KB * 128, 64, grow);
                        tma_load_2d(&tmGl, full + s, st + L::OP_BYTES, 0, grow);
                        tma_load_2d(&tmGl, full + s, st + L::OP_BYTES + L::KB * 128, 64, grow);
                        const int kc0 = ((2 * h) * K + kk) * BK, kc1 = ((2 * h + 1) * K + kk) * BK;   // the chunk's two channel blocks
                        tma_load_2d(&tmWh, full + s, st + 2 * L::OP_BYTES, kc0, kb * L::KB);
                        tma_load_2d(&tmWh, full + s, st + 2 * L::OP_BYTES + L::KB * 128, kc1, kb * L::KB);
                        tma_load_2d(&tmWl, full + s, st + 3 * L::OP_BYTES, kc0, kb * L::KB);
                        tma_load_2d(&tmWl, full + s, st + 3 * L::OP_BYTES + L::KB * 128, kc1, kb * L::KB);
                    }
        }
    } else if (warp >= 2 && threadIdx.x < 64 + kProducerThreads) {
        // Epilogue warp = (row quarter q, slice `part`).  It drains 32 channels of its quarter's 32 pixel rows into the shared staging tile
        // and then owns 8 of those rows for all 128 channels (8 lanes per row, 2 rows per lane: the forward's gather mapping), so the sums
        // over channels stay in registers.  Only the four warps of a quarter synchronise (named barriers 1 + q and 5 + q); the quarters
        // drift apart, which overlaps one quarter's gather latency with another's arithmetic.
        const int pwp = warp - 2;
        const int q = warp & 3, part = pwp >> 2;
        const int sub = lane >> 3, j = lane & 7;
        const uint32_t stg = smem_u32(smem + L::STG_OFF);
        const float *xb = a.xh + (int64_t)b * a.H * a.W * a.C + j * 4;
        float *gxb = a.gxh ? a.gxh + (int64_t)b * a.H * a.W * a.C + j * 4 : nullptr;
        const int R0 = q * 32;
        int rrow[2];
#pragma unroll
        for (int u = 0; u < 2; ++u) rrow[u] = R0 + part * 8 + u * 4 + sub;
        if (part == 0 && (int)blockIdx.y < K)
            dcn_dgrad_store_row(a, tab_of(0), dcn_dgrad_load_row(a, b, blockIdx.y, R0 + lane, ty0, tx0), blockIdx.y, R0 + lane, ty0, tx0);
        int n = 0, t = 0;
        for (int kk = blockIdx.y; kk < K; kk += a.tap_splits, ++t) {
            const int tb = t & 1;
            const DcnDTab T = tab_of(tb);
            float vh[2] = {0.f, 0.f}, vw[2] = {0.f, 0.f}, vm[2] = {0.f, 0.f};
            for (int h = 0; h < a.nch; ++h, ++n) {
                const int buf = n & 1;
                mbar_wait(acc_full + buf, (n >> 1) & 1);
                {
                    uint32_t rr[32];
                    acc_ld<32>(acc_tile, AccTile<BN>::LD, q * 32, part * 32, rr);
                    const int r = R0 + lane;
                    const uint32_t rb = stg + (uint32_t)r * 512u;
#pragma unroll
                    for (int c4 = 0; c4 < 8; ++c4)
                        asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(rb + ((((uint32_t)(part * 8 + c4)) ^ (uint32_t)(r & 31)) << 4)),
                                     "r"(rr[4 * c4]), "r"(rr[4 * c4 + 1]), "r"(rr[4 * c4 + 2]), "r"(rr[4 * c4 + 3]) : "memory");
                }
                asm volatile("bar.sync %0, 128;" ::"r"(1 + q) : "memory");
                if (lane == 0) mbar_arrive_cta(acc_empty + buf);
                // the next tap's table: its three global loads are issued now and consumed after this N block's work
                const bool prep = part == 0 && h == 0 && kk + a.tap_splits < K;
                DcnDRaw raw = {0.f, 0.f, 0.f};
                if (prep) raw = dcn_dgrad_load_row(a, b, kk + a.tap_splits, R0 + lane, ty0, tx0);
#pragma unroll
                for (int u = 0; u < 2; ++u) {
                    const int r = rrow[u];
                    const float4 w = T.w[r], ch = T.h[r], cv = T.v[r];
                    const uint2 cc = T.c[r];
                    const float mk = T.m[r];               // ch / cv carry the mask already; the scatter needs it separately
                    const int y0 = (int)(cc.x & 0xffffu) * a.W, y1 = (int)(cc.x >> 16) * a.W;
                    const int x0 = (int)(cc.y & 0xffffu), x1 = (int)(cc.y >> 16);
                    const int64_t o1 = (int64_t)(y0 + x0) * a.C + h * 128, o2 = (int64_t)(y0 + x1) * a.C + h * 128;
                    const int64_t o3 = (int64_t)(y1 + x0) * a.C + h * 128, o4 = (int64_t)(y1 + x1) * a.C + h * 128;
#pragma unroll 1
                    for (int eh = 0; eh < 4; eh += 2) {         // two 16-byte channel chunks at a time (register budget: 96)
                        float4 g[2], v1[2], v2[2], v3[2], v4[2];
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            v1[e] = __ldg(reinterpret_cast<const float4 *>(xb + o1) + (eh + e) * 8);
                            v2[e] = __ldg(reinterpret_cast<const float4 *>(xb + o2) + (eh + e) * 8);
                            v3[e] = __ldg(reinterpret_cast<const float4 *>(xb + o3) + (eh + e) * 8);
                            v4[e] = __ldg(reinterpret_cast<const float4 *>(xb + o4) + (eh + e) * 8);
                            const uint32_t ad = stg + (uint32_t)r * 512u + ((((uint32_t)(j + 8 * (eh + e))) ^ (uint32_t)(r & 31)) << 4);
                            asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(g[e].x), "=f"(g[e].y), "=f"(g[e].z), "=f"(g[e].w) : "r"(ad));
                        }
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
#define MR_DCN_CH(F)                                                                                              \
                            {                                                                                         \
                                const float gg = g[e].F;                                                              \
                                vm[u] = fmaf(gg, w.x * v1[e].F + w.y * v2[e].F + w.z * v3[e].F + w.w * v4[e].F, vm[u]);      \
                                vh[u] = fmaf(gg, ch.x * v1[e].F + ch.y * v2[e].F + ch.z * v3[e].F + ch.w * v4[e].F, vh[u]);  \
                                vw[u] = fmaf(gg, cv.x * v1[e].F + cv.y * v2[e].F + cv.z * v3[e].F + cv.w * v4[e].F, vw[u]);  \
                            }
                            MR_DCN_CH(x) MR_DCN_CH(y) MR_DCN_CH(z) MR_DCN_CH(w)
#undef MR_DCN_CH
                            if (gxb) {
                                const float gx = g[e].x * mk, gy = g[e].y * mk, gz = g[e].z * mk, gw = g[e].w * mk;
                                const int eo = (eh + e) * 32;
                                if (w.x != 0.f) red_add_v4(gxb + o1 + eo, w.x * gx, w.x * gy, w.x * gz, w.x * gw);
                                if (w.y != 0.f) red_add_v4(gxb + o2 + eo, w.y * gx, w.y * gy, w.y * gz, w.y * gw);
                                if (w.z != 0.f) red_add_v4(gxb + o3 + eo, w.z * gx, w.z * gy, w.z * gz, w.z * gw);
                                if (w.w != 0.f) red_add_v4(gxb + o4 + eo, w.w * gx, w.w * gy, w.w * gz, w.w * gw);
                            }
                        }
                    }
                }
                if (prep) dcn_dgrad_store_row(a, tab_of(tb ^ 1), raw, kk + a.tap_splits, R0 + lane, ty0, tx0);
                asm volatile("bar.sync %0, 128;" ::"r"(5 + q) : "memory");
            }
            // the tap is complete: fold the 8 channel lanes of each pixel row and write its three gradients
#pragma unroll
            for (int u = 0; u < 2; ++u) {
#pragma unroll
                for (int sft = 1; sft < 8; sft <<= 1) {
                    vh[u] += __shfl_xor_sync(0xffffffffu, vh[u], sft);
                    vw[u] += __shfl_xor_sync(0xffffffffu, vw[u], sft);
                    vm[u] += __shfl_xor_sync(0xffffffffu, vm[u], sft);
                }
                const int r = rrow[u];
                const int py = ty0 + (r >> 4), px = tx0 + (r & 15);
                if (j == 0 && py < a.Ho && px < a.Wo) {
                    const int pc = py * a.Wo + px;
                    if (a.goff) {
                        float *gp = a.goff + (int64_t)b * a.goff_bs;
                        gp[(int64_t)(2 * kk) * a.P + pc] = vh[u];
                        gp[(int64_t)(2 * kk + 1) * a.P + pc] = vw[u];
                    }
                    if (a.gmask) a.gmask[(int64_t)b * a.gmask_bs + (int64_t)kk * a.P + pc] = vm[u];
                }
            }
        }
    }
}

// y [B][C][P] += x [B][P][C]   (the NHWC gradient scratch folded into the caller's NCHW grad_input, which is accumulated into)
__global__ void __launch_bounds__(256) dcn_nhwc_to_nchw_add_kernel(const float *__restrict__ x, float *__restrict__ y, int C, int P) {
    __shared__ float t[32][33];
    const int b = blockIdx.z, p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    for (int i = ty; i < 32; i += 8) {
        const int p = p0 + i, c = c0 + tx;
        t[i][tx] = (p < P && c < C) ? x[((int64_t)b * P + p) * C + c] : 0.f;
    }
    __syncthreads();
    for (int i = ty; i < 32; i += 8) {
        const int c = c0 + i, p = p0 + tx;
        if (p < P && c < C) y[((int64_t)b * C + c) * P + p] += t[tx][i];
    }
}

// grad_output [B][Cout][P] fp32 -> hi / lo bf16 [B * tiles][Cout][128] in the 8 x 16 tile order of the kernels (0 outside the map)
__global__ void dcn_go_retile_kernel(const float *__restrict__ go, int B, int Cout, int Ho, int Wo, int tiles_x, int tiles_per_sample,
                                     bf16 *__restrict__ hi, bf16 *__restrict__ lo) {
    // one thread = one 16-pixel tile row of one channel: 64 contiguous bytes in, 32 + 32 contiguous bytes out
    const int64_t n = (int64_t)B * tiles_per_sample * Cout * 8;
    const bool vec = (Wo & 3) == 0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int gr = (int)(i & 7);
        int64_t t = i >> 3;
        const int co = (int)(t % Cout); t /= Cout;
        const int tile = (int)(t % tiles_per_sample);
        const int b = (int)(t / tiles_per_sample);
        const int py = (tile / tiles_x) * 8 + gr, px0 = (tile % tiles_x) * 16;
        float v[16];
        const float *src = go + ((int64_t)b * Cout + co) * Ho * Wo + (int64_t)py * Wo + px0;
        if (py < Ho && vec && px0 + 16 <= Wo) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float4 f = __ldg(reinterpret_cast<const float4 *>(src) + e);
                v[4 * e] = f.x; v[4 * e + 1] = f.y; v[4 * e + 2] = f.z; v[4 * e + 3] = f.w;
            }
        } else {
#pragma unroll
            for (int e = 0; e < 16; ++e) v[e] = (py < Ho && px0 + e < Wo) ? __ldg(src + e) : 0.f;
        }
        uint32_t ph[8], pl[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            const __nv_bfloat162 h2 = __floats2bfloat162_rn(v[2 * e], v[2 * e + 1]);
            const float2 f = __bfloat1622float2(h2);
            const __nv_bfloat162 l2 = __floats2bfloat162_rn(v[2 * e] - f.x, v[2 * e + 1] - f.y);
            ph[e] = *reinterpret_cast<const uint32_t *>(&h2);
            pl[e] = *reinterpret_cast<const uint32_t *>(&l2);
        }
        uint4 *dh = reinterpret_cast<uint4 *>(hi + i * 16), *dl = reinterpret_cast<uint4 *>(lo + i * 16);
        dh[0] = make_uint4(ph[0], ph[1], ph[2], ph[3]); dh[1] = make_uint4(ph[4], ph[5], ph[6], ph[7]);
        dl[0] = make_uint4(pl[0], pl[1], pl[2], pl[3]); dl[1] = make_uint4(pl[4], pl[5], pl[6], pl[7]);
    }
}

// x [B][C][P] -> y [B][P][C] (fp32), 32 x 32 tiles through shared memory; both sides 128-byte rows
__global__ void __launch_bounds__(256)
dcn_nchw_to_nhwc_kernel(const float *__restrict__ x, float *__restrict__ y, int C, int P) {
    __shared__ float tile[32][33];
    const int b = blockIdx.z, c0 = blockIdx.y * 32, p0 = blockIdx.x * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const float *xb = x + (int64_t)b * C * P;
    float *yb = y + (int64_t)b * C * P;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int c = c0 + ty + 8 * j, p = p0 + tx;
        tile[ty + 8 * j][tx] = (c < C && p < P) ? __ldg(xb + (int64_t)c * P + p) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int p = p0 + ty + 8 * j, c = c0 + tx;
        if (p < P && c < C) yb[(int64_t)p * C + c] = tile[tx][ty + 8 * j];
    }
}

// weight [Cout][C][K] fp32 -> hi / lo bf16 [Cout][(cb * K + k) * 64 + cl]  (channel c = cb * 64 + cl)
__global__ void dcn_weight_pack_kernel(const float *__restrict__ w, int Cout, int C, int K, bf16 *__restrict__ hi, bf16 *__restrict__ lo) {
    const int64_t n = (int64_t)Cout * C * K;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        // i = co * (C*K) + (cb * K + k) * 64 + cl   with channel c = cb * 64 + cl
        const int cl = (int)(i % 64);
        int64_t t = i / 64;
        const int k = (int)(t % K); t /= K;
        const int cb = (int)(t % (C / 64));
        const int co = (int)(t / (C / 64));
        const int c = cb * 64 + cl;
        const float v = w[((int64_t)co * C + c) * K + k];
        const bf16 h = __float2bfloat16_rn(v);
        hi[i] = h;
        lo[i] = __float2bfloat16_rn(v - __bfloat162float(h));
    }
}

// launch of the fused weight gradient once the NHWC input and the re-tiled grad_output exist
int launch_dcn_wgrad(DcnWArgs &a, const bf16 *ghi, const bf16 *glo, cudaStream_t st) {
    CUtensorMap th, tl;
    int rc = make_map(&th, ghi, BM, (int64_t)a.ntiles * a.Cout, BM, BK, BM);
    if (rc) return rc;
    rc = make_map(&tl, glo, BM, (int64_t)a.ntiles * a.Cout, BM, BK, BM);
    if (rc) return rc;
    // split-K over the pixel tiles: whole waves of CTAs (one CTA per SM), the fewest (rounds x tiles per CTA + per-CTA overhead)
    const int ctas_fixed = a.nkb * (a.Cout / BM);
    int splits = 1;
    int64_t best = -1;
    for (int waves = 1; waves <= 4; ++waves) {
        int sp = (int)((int64_t)waves * sm_count() / ctas_fixed);
        sp = sp < 1 ? 1 : (sp > a.ntiles ? a.ntiles : sp);
        const int64_t rounds = ceil_div((int64_t)ctas_fixed * sp, sm_count());
        const int64_t cost = rounds * (ceil_div(a.ntiles, sp) + 3);
        if (best < 0 || cost < best) { best = cost; splits = sp; }
    }
    a.splits = splits;
    { int rc_attr = ensure_dyn_smem((const void *)dcn_wgrad_tcgen05_kernel, DcnWSmem::TOTAL, "dcn_wgrad_tcgen05 smem attr"); if (rc_attr) return rc_attr; }
    dim3 grid((unsigned)a.nkb, (unsigned)splits, (unsigned)(a.Cout / BM));
    dcn_wgrad_tcgen05_kernel<<<grid, kDcnThreads, DcnWSmem::TOTAL, st>>>(th, tl, a);
    return check_launch("dcn_wgrad_tcgen05_kernel");
}

template <int BN, int STAGES>
int launch_dcn_fwd(const CUtensorMap &th, const CUtensorMap &tl, const DcnFArgs &a, cudaStream_t st) {
    using L = DcnSmem<BN, STAGES>;
    auto kern = dcn_fwd_tcgen05_kernel<BN, STAGES>;
    const int smem = L::total(a.kh * a.kw);
    if (smem > 227 * 1024) return MR_ERR_UNSUPPORTED;
    { int rc_attr = ensure_dyn_smem((const void *)kern, smem, "dcn_fwd_tcgen05 smem attr"); if (rc_attr) return rc_attr; }
    dim3 grid((unsigned)(a.B * a.tiles_per_sample), (unsigned)(a.Cout / BN), 1);
    kern<<<grid, kDcnThreads, smem, st>>>(th, tl, a);
    return check_launch("dcn_fwd_tcgen05_kernel");
}

}  // namespace

extern "C" {

/* scratch the fused forward needs: NHWC copy of the input + hi/lo packed weights (256-byte aligned pieces) */
int64_t mr_dcn_fused_workspace_bytes(int64_t B, int64_t C, int64_t H, int64_t W, int64_t Cout, int64_t kh, int64_t kw) {
    const int64_t x = round_up(B * H * W * C * 4, 256);
    const int64_t w = round_up(Cout * C * kh * kw * 2, 256);
    return x + 2 * w;
}

/* MR_ERR_UNSUPPORTED when the shape is outside the fused path (the caller then runs the unfused kernels of dcn.cu). */
int mr_dcn_forward_fused_f32(const float *input, const float *weight, const float *bias, const float *offset,
                             int64_t offset_bstride, const float *mask, int64_t mask_bstride, float *output,
                             float *workspace, int64_t workspace_bytes, int B, int C, int H, int W, int Cout, int kh, int kw,
                             int sh, int sw, int ph, int pw, int dh, int dw, int group, int dg, void *stream) {
    if (group != 1 || dg != 1 || C % 64 || Cout % 128 || B <= 0 || H > 65535 || W > 65535) return MR_ERR_UNSUPPORTED;
    if (getenv("MR_DCN_UNFUSED")) return MR_ERR_UNSUPPORTED;
    if (!input || !weight || !offset || !output || !workspace) return MR_ERR_NULL_POINTER;
    if (workspace_bytes < mr_dcn_fused_workspace_bytes(B, C, H, W, Cout, kh, kw) || ((uintptr_t)workspace % 256)) return MR_ERR_UNSUPPORTED;
    DcnFArgs a;
    a.B = B; a.C = C; a.H = H; a.W = W; a.Cout = Cout; a.kh = kh; a.kw = kw; a.sh = sh; a.sw = sw; a.ph = ph; a.pw = pw;
    a.dh = dh; a.dw = dw;
    a.Ho = (H + 2 * ph - (dh * (kh - 1) + 1)) / sh + 1;
    a.Wo = (W + 2 * pw - (dw * (kw - 1) + 1)) / sw + 1;
    if (a.Ho <= 0 || a.Wo <= 0) return MR_ERR_BAD_SHAPE;
    a.P = a.Ho * a.Wo;
    a.tiles_x = (int)ceil_div(a.Wo, 16);
    a.tiles_per_sample = a.tiles_x * (int)ceil_div(a.Ho, 8);
    a.ncb = C / BK; a.nkb = kh * kw * a.ncb;
    if ((int64_t)B * a.tiles_per_sample > 0x7fffffffLL) return MR_ERR_UNSUPPORTED;
    cudaStream_t st = (cudaStream_t)stream;
    unsigned char *ws = (unsigned char *)workspace;
    float *xh = (float *)ws;
    const int64_t xbytes = round_up((int64_t)B * H * W * C * 4, 256), wbytes = round_up((int64_t)Cout * C * kh * kw * 2, 256);
    bf16 *whi = (bf16 *)(ws + xbytes), *wlo = (bf16 *)(ws + xbytes + wbytes);
    {
        dim3 tg((unsigned)ceil_div((int64_t)H * W, 32), (unsigned)ceil_div(C, 32), (unsigned)B);
        dcn_nchw_to_nhwc_kernel<<<tg, 256, 0, st>>>(input, xh, C, H * W);
    }
    int rc = check_launch("dcn_nchw_to_nhwc_kernel");
    if (rc) return rc;
    const int64_t nw = (int64_t)Cout * C * kh * kw;
    dcn_weight_pack_kernel<<<(unsigned)std::min<int64_t>(ceil_div(nw, 256), sm_count() * 8), 256, 0, st>>>(weight, Cout, C, kh * kw, whi, wlo);
    rc = check_launch("dcn_weight_pack_kernel");
    if (rc) return rc;
    a.xh = xh; a.off = offset; a.msk = mask; a.bias = bias; a.out = output; a.off_bs = offset_bstride; a.mask_bs = mask_bstride;
    const int64_t Kt = (int64_t)kh * kw * C;
    CUtensorMap th, tl;
    rc = make_map(&th, whi, Kt, Cout, Kt, BK, 128);
    if (rc) return rc;
    rc = make_map(&tl, wlo, Kt, Cout, Kt, BK, 128);
    if (rc) return rc;
    /* two stages, not three: the 64 KB saved become L1 for the gathers (MR_DCN_STAGES3 selects three for experiments) */
    static const bool three = getenv("MR_DCN_STAGES3") != nullptr;
    if (three) return launch_dcn_fwd<128, 3>(th, tl, a, st);
    return launch_dcn_fwd<128, 2>(th, tl, a, st);
}

/* scratch of the fused backward: NHWC copies of the input and of grad_input, re-tiled hi / lo grad_output, packed hi / lo weights */
int64_t mr_dcn_fused_backward_workspace_bytes(int64_t B, int64_t C, int64_t H, int64_t W, int64_t Cout, int64_t Ho, int64_t Wo,
                                              int64_t kh, int64_t kw) {
    const int64_t tiles = ceil_div(Wo, 16) * ceil_div(Ho, 8);
    return 2 * round_up(B * H * W * C * 4, 256) + 2 * round_up(B * tiles * Cout * BM * 2, 256) + 2 * round_up(Cout * C * kh * kw * 2, 256);
}

/* The whole of mr_dcn_backward_f32 except grad_bias on the fused kernels (weight gradient + data gradient); MR_ERR_UNSUPPORTED
 * outside group = deformable_group = 1, C % 128 == 0, Cout % 128 == 0 or when the workspace is too small. */
int mr_dcn_backward_fused_f32(const float *input, const float *weight, const float *offset, int64_t offset_bstride, const float *mask,
                              int64_t mask_bstride, const float *grad_output, float *grad_input, float *grad_weight,
                              float *grad_offset, int64_t grad_offset_bstride, float *grad_mask, int64_t grad_mask_bstride,
                              float weight_grad_scale, float *workspace, int64_t workspace_bytes, int B, int C, int H, int W, int Cout,
                              int kh, int kw, int sh, int sw, int ph, int pw, int dh, int dw, int group, int dg, void *stream) {
    if (group != 1 || dg != 1 || C % 128 || Cout % 128 || B <= 0 || H > 65535 || W > 65535) return MR_ERR_UNSUPPORTED;
    if (getenv("MR_DCN_UNFUSED") || getenv("MR_DCN_UNFUSED_DGRAD")) return MR_ERR_UNSUPPORTED;
    if (!input || !weight || !offset || !grad_output || !workspace) return MR_ERR_NULL_POINTER;
    const int Ho = (H + 2 * ph - (dh * (kh - 1) + 1)) / sh + 1, Wo = (W + 2 * pw - (dw * (kw - 1) + 1)) / sw + 1;
    if (Ho <= 0 || Wo <= 0) return MR_ERR_BAD_SHAPE;
    if (workspace_bytes < mr_dcn_fused_backward_workspace_bytes(B, C, H, W, Cout, Ho, Wo, kh, kw) || ((uintptr_t)workspace % 256)) return MR_ERR_UNSUPPORTED;
    const int tiles_x = (int)ceil_div(Wo, 16), tiles_per_sample = tiles_x * (int)ceil_div(Ho, 8), ntiles = B * tiles_per_sample;
    if ((int64_t)ntiles * Cout > 0x7fffffffLL) return MR_ERR_UNSUPPORTED;
    cudaStream_t st = (cudaStream_t)stream;
    unsigned char *ws = (unsigned char *)workspace;
    const int64_t xbytes = round_up((int64_t)B * H * W * C * 4, 256), gbytes = round_up((int64_t)ntiles * Cout * BM * 2, 256);
    const int64_t wbytes = round_up((int64_t)Cout * C * kh * kw * 2, 256);
    float *xh = (float *)ws, *gxh = (float *)(ws + xbytes);
    bf16 *ghi = (bf16 *)(ws + 2 * xbytes), *glo = (bf16 *)(ws + 2 * xbytes + gbytes);
    bf16 *whi = (bf16 *)(ws + 2 * xbytes + 2 * gbytes), *wlo = (bf16 *)(ws + 2 * xbytes + 2 * gbytes + wbytes);
    const bool want_data = grad_input || grad_offset || grad_mask;
    if (!want_data && !grad_weight) return MR_OK;
    {
        dim3 tg((unsigned)ceil_div((int64_t)H * W, 32), (unsigned)ceil_div(C, 32), (unsigned)B);
        dcn_nchw_to_nhwc_kernel<<<tg, 256, 0, st>>>(input, xh, C, H * W);
    }
    int rc = check_launch("dcn_nchw_to_nhwc_kernel");
    if (rc) return rc;
    const int64_t ng = (int64_t)ntiles * Cout * 8;
    dcn_go_retile_kernel<<<(unsigned)std::min<int64_t>(ceil_div(ng, 256), (int64_t)sm_count() * 16), 256, 0, st>>>(
        grad_output, B, Cout, Ho, Wo, tiles_x, tiles_per_sample, ghi, glo);
    rc = check_launch("dcn_go_retile_kernel");
    if (rc) return rc;
    if (grad_weight) {
        DcnWArgs a;
        a.B = B; a.C = C; a.H = H; a.W = W; a.Cout = Cout; a.kh = kh; a.kw = kw; a.sh = sh; a.sw = sw; a.ph = ph; a.pw = pw; a.dh = dh; a.dw = dw;
        a.Ho = Ho; a.Wo = Wo; a.P = Ho * Wo; a.tiles_x = tiles_x; a.tiles_per_sample = tiles_per_sample; a.ncb = C / BK; a.nkb = kh * kw * a.ncb;
        a.ntiles = ntiles;
        a.xh = xh; a.off = offset; a.msk = mask; a.off_bs = offset_bstride; a.mask_bs = mask_bstride; a.gw = grad_weight; a.scale = weight_grad_scale;
        rc = launch_dcn_wgrad(a, ghi, glo, st);
        if (rc) return rc;
    }
    if (want_data) {
        const int64_t nw = (int64_t)Cout * C * kh * kw;
        dcn_weight_pack_kernel<<<(unsigned)std::min<int64_t>(ceil_div(nw, 256), sm_count() * 8), 256, 0, st>>>(weight, Cout, C, kh * kw, whi, wlo);
        rc = check_launch("dcn_weight_pack_kernel");
        if (rc) return rc;
        if (grad_input) MR_CUDA_TRY(cudaMemsetAsync(gxh, 0, (size_t)B * H * W * C * 4, st), "cudaMemsetAsync(dcn grad_input scratch)");
        DcnDArgs a;
        a.B = B; a.C = C; a.H = H; a.W = W; a.Cout = Cout; a.kh = kh; a.kw = kw; a.sh = sh; a.sw = sw; a.ph = ph; a.pw = pw; a.dh = dh; a.dw = dw;
        a.Ho = Ho; a.Wo = Wo; a.P = Ho * Wo; a.tiles_x = tiles_x; a.tiles_per_sample = tiles_per_sample; a.nch = C / 128; a.nkk = Cout / DcnDSmem::KB;
        a.xh = xh; a.off = offset; a.msk = mask; a.gxh = grad_input ? gxh : nullptr; a.goff = grad_offset; a.gmask = grad_mask;
        a.off_bs = offset_bstride; a.mask_bs = mask_bstride; a.goff_bs = grad_offset_bstride; a.gmask_bs = grad_mask_bstride;
        const int K = kh * kw;
        // taps are spread over grid.y (a divisor of the tap count): the fewest (rounds of CTAs x N blocks per CTA + per-CTA overhead)
        int splits = 1;
        int64_t best = -1;
        for (int sp = 1; sp <= K; ++sp) {
            if (K % sp) continue;
            const int64_t cost = ceil_div((int64_t)ntiles * sp, sm_count()) * ((int64_t)(K / sp) * a.nch + 1);
            if (best < 0 || cost < best) { best = cost; splits = sp; }
        }
        a.tap_splits = splits;
        CUtensorMap gh, gl, wh, wl;
        const int64_t Kt = (int64_t)K * C;
        if ((rc = make_map(&gh, ghi, BM, (int64_t)ntiles * Cout, BM, BK, DcnDSmem::KB))) return rc;
        if ((rc = make_map(&gl, glo, BM, (int64_t)ntiles * Cout, BM, BK, DcnDSmem::KB))) return rc;
        if ((rc = make_map(&wh, whi, Kt, Cout, Kt, BK, DcnDSmem::KB))) return rc;
        if ((rc = make_map(&wl, wlo, Kt, Cout, Kt, BK, DcnDSmem::KB))) return rc;
        { int rc_attr = ensure_dyn_smem((const void *)dcn_dgrad_tcgen05_kernel, DcnDSmem::TOTAL, "dcn_dgrad_tcgen05 smem attr"); if (rc_attr) return rc_attr; }
        dim3 grid((unsigned)ntiles, (unsigned)splits);
        dcn_dgrad_tcgen05_kernel<<<grid, kDcnThreads, DcnDSmem::TOTAL, st>>>(gh, gl, wh, wl, a);
        rc = check_launch("dcn_dgrad_tcgen05_kernel");
        if (rc) return rc;
        if (grad_input) {
            dim3 tg((unsigned)ceil_div((int64_t)H * W, 32), (unsigned)ceil_div(C, 32), (unsigned)B);
            dcn_nhwc_to_nchw_add_kernel<<<tg, 256, 0, st>>>(gxh, grad_input, C, H * W);
            rc = check_launch("dcn_nhwc_to_nchw_add_kernel");
            if (rc) return rc;
        }
    }
    return MR_OK;
}

/* scratch of the fused weight gradient: NHWC copy of the input + re-tiled hi / lo grad_output */
int64_t mr_dcn_fused_wgrad_workspace_bytes(int64_t B, int64_t C, int64_t H, int64_t W, int64_t Cout, int64_t Ho, int64_t Wo) {
    const int64_t tiles = ceil_div(Wo, 16) * ceil_div(Ho, 8);
    return round_up(B * H * W * C * 4, 256) + 2 * round_up(B * tiles * Cout * BM * 2, 256);
}

/* grad_weight [Cout][C][kh*kw] += scale * (grad_output (*) deformable columns); MR_ERR_UNSUPPORTED outside the fused path. */
int mr_dcn_wgrad_fused_f32(const float *input, const float *offset, int64_t offset_bstride, const float *mask, int64_t mask_bstride,
                           const float *grad_output, float *grad_weight, float scale, float *workspace, int64_t workspace_bytes,
                           int B, int C, int H, int W, int Cout, int kh, int kw, int sh, int sw, int ph, int pw, int dh, int dw,
                           int group, int dg, void *stream) {
    if (group != 1 || dg != 1 || C % 64 || Cout % 128 || B <= 0 || H > 65535 || W > 65535) return MR_ERR_UNSUPPORTED;
    if (getenv("MR_DCN_UNFUSED") || getenv("MR_DCN_UNFUSED_WGRAD")) return MR_ERR_UNSUPPORTED;
    if (!input || !offset || !grad_output || !grad_weight || !workspace) return MR_ERR_NULL_POINTER;
    DcnWArgs a;
    a.B = B; a.C = C; a.H = H; a.W = W; a.Cout = Cout; a.kh = kh; a.kw = kw; a.sh = sh; a.sw = sw; a.ph = ph; a.pw = pw;
    a.dh = dh; a.dw = dw;
    a.Ho = (H + 2 * ph - (dh * (kh - 1) + 1)) / sh + 1;
    a.Wo = (W + 2 * pw - (dw * (kw - 1) + 1)) / sw + 1;
    if (a.Ho <= 0 || a.Wo <= 0) return MR_ERR_BAD_SHAPE;
    if (workspace_bytes < mr_dcn_fused_wgrad_workspace_bytes(B, C, H, W, Cout, a.Ho, a.Wo) || ((uintptr_t)workspace % 256)) return MR_ERR_UNSUPPORTED;
    a.P = a.Ho * a.Wo;
    a.tiles_x = (int)ceil_div(a.Wo, 16);
    a.tiles_per_sample = a.tiles_x * (int)ceil_div(a.Ho, 8);
    a.ncb = C / BK; a.nkb = kh * kw * a.ncb;
    a.ntiles = B * a.tiles_per_sample;
    if ((int64_t)a.ntiles * Cout > 0x7fffffffLL) return MR_ERR_UNSUPPORTED;
    cudaStream_t st = (cudaStream_t)stream;
    unsigned char *ws = (unsigned char *)workspace;
    float *xh = (float *)ws;
    const int64_t xbytes = round_up((int64_t)B * H * W * C * 4, 256), gbytes = round_up((int64_t)a.ntiles * Cout * BM * 2, 256);
    bf16 *ghi = (bf16 *)(ws + xbytes), *glo = (bf16 *)(ws + xbytes + gbytes);
    {
        dim3 tg((unsigned)ceil_div((int64_t)H * W, 32), (unsigned)ceil_div(C, 32), (unsigned)B);
        dcn_nchw_to_nhwc_kernel<<<tg, 256, 0, st>>>(input, xh, C, H * W);
    }
    int rc = check_launch("dcn_nchw_to_nhwc_kernel");
    if (rc) return rc;
    const int64_t ng = (int64_t)a.ntiles * Cout * 8;
    dcn_go_retile_kernel<<<(unsigned)std::min<int64_t>(ceil_div(ng, 256), (int64_t)sm_count() * 16), 256, 0, st>>>(
        grad_output, B, Cout, a.Ho, a.Wo, a.tiles_x, a.tiles_per_sample, ghi, glo);
    rc = check_launch("dcn_go_retile_kernel");
    if (rc) return rc;
    a.xh = xh; a.off = offset; a.msk = mask; a.off_bs = offset_bstride; a.mask_bs = mask_bstride; a.gw = grad_weight; a.scale = scale;
    return launch_dcn_wgrad(a, ghi, glo, st);
}

}  // extern "C"
