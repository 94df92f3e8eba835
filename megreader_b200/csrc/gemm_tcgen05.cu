// Hopper dense GEMM: bf16 operands, fp32 accumulation in the registers of one MMA warpgroup (wgmma.mma_async m64nBNk16,
// two per K step for the 128-row tile), operands staged by TMA (cp.async.bulk.tensor, 128-byte swizzle) through a
// 3..8-stage mbarrier ring.
//
//   C[M,N] (row-major, bf16 or fp32)  (+)=  op(A)[M,K] * op(B)[K,N]
//     A_MN = 0: A stored [M,K] row-major (K-major operand)        A_MN = 1: A stored [K,M] row-major (MN-major operand)
//     B_MN = 0: B stored [N,K] row-major (K-major operand)        B_MN = 1: B stored [K,N] row-major (MN-major operand)
//   i.e. (0,0) is the "NT" form used for conv forward / dgrad / Linear layers, (1,1) is the "TN" form of weight
//   gradients  dW[Cout, K] = dZ[P, Cout]^T * col[P, K].
//   Epilogue: optional per-column bias, optional ReLU, fp32 or bf16 store, or fp32 atomic accumulation (split-K).
//
// Warp roles (384 threads): warp 0 = TMA producer (one elected lane), warps 2..5 = epilogue (one accumulator row per
// thread -> global), warps 8..11 = the MMA warpgroup, which hands the finished accumulator to the epilogue warps through
// a shared-memory tile laid over the drained operand ring.  One 128 x BN output tile (BN <= 128: the accumulator is
// BN registers per MMA thread) per CTA (grid = tiles x split-K); K loops over 64-element blocks.
#include "wgmma.cuh"
#include <stdlib.h>

namespace {

struct GemmArgs {
    int M, N, K;
    int64_t ldc;
    void *C;
    const float *bias;
    int relu, out_bf16, atomic;     // atomic: fp32 atomicAdd into C (split-K)
    int kblocks_per_split;
};

// Epilogue shared by the GEMM and convolution kernels: warps 2..5, accumulator tile -> registers -> (bias, ReLU) -> global.
template <int BN>
__device__ __forceinline__ void epilogue_store(const GemmArgs &g, const float *acc, uint64_t *tmem_full, int m0, int n0,
                                               int warp, int lane, bool have_acc, int64_t row_override = -2) {
        const int q = warp & 3;                               // 32-row quarter of the tile this warp stores
        // output row of this thread: m0 + tile row, or an explicit row (-1 = none) for tiles that are not row ranges
        const int64_t row = row_override == -2 ? (int64_t)(m0 + q * 32 + lane) : (row_override < 0 ? (int64_t)g.M : row_override);
        const int nkb = have_acc ? 1 : 0;
        if (nkb > 0) {
            mbar_wait(tmem_full, 0);
        }
        float *Cf = (float *)g.C;
        bf16 *Ch = (bf16 *)g.C;
#pragma unroll 1
        for (int c = 0; c < BN / 32; ++c) {
            uint32_t r[32];
            if (nkb > 0) acc_ld<32>(acc, AccTile<BN>::LD, q * 32, c * 32, r);
            else {
#pragma unroll
                for (int j = 0; j < 32; ++j) r[j] = 0;
            }
            const int nbase = n0 + c * 32;
            if (row < g.M && nbase < g.N) {
                float v[32];
#pragma unroll
                for (int j = 0; j < 32; ++j) {
                    v[j] = __uint_as_float(r[j]);
                    if (g.bias && nbase + j < g.N) v[j] += g.bias[nbase + j];
                    if (g.relu) v[j] = fmaxf(v[j], 0.f);
                }
                const bool full32 = nbase + 32 <= g.N;
                if (g.atomic) {
                    float *dst = Cf + (int64_t)row * g.ldc + nbase;
#pragma unroll
                    for (int j = 0; j < 32; ++j)
                        if (full32 || nbase + j < g.N) atomicAdd(dst + j, v[j]);
                } else if (g.out_bf16) {
                    bf16 *dst = Ch + (int64_t)row * g.ldc + nbase;
                    if (full32 && ((uintptr_t)dst % 16 == 0)) {
#pragma unroll
                        for (int j = 0; j < 32; j += 8) {
                            uint4 pk;
                            __nv_bfloat162 *h = reinterpret_cast<__nv_bfloat162 *>(&pk);
#pragma unroll
                            for (int e = 0; e < 4; ++e) h[e] = __floats2bfloat162_rn(v[j + 2 * e], v[j + 2 * e + 1]);
                            *reinterpret_cast<uint4 *>(dst + j) = pk;
                        }
                    } else {
#pragma unroll
                        for (int j = 0; j < 32; ++j)
                            if (nbase + j < g.N) dst[j] = __float2bfloat16_rn(v[j]);
                    }
                } else {
                    float *dst = Cf + (int64_t)row * g.ldc + nbase;
                    if (full32 && ((uintptr_t)dst % 16 == 0)) {
#pragma unroll
                        for (int j = 0; j < 32; j += 4) *reinterpret_cast<float4 *>(dst + j) = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
                    } else {
#pragma unroll
                        for (int j = 0; j < 32; ++j)
                            if (nbase + j < g.N) dst[j] = v[j];
                    }
                }
            }
        }
}

constexpr int kGemmMma0 = 256;                      // first thread of the MMA warpgroup (warps 6, 7 are padding)
constexpr int kGemmThreads = kGemmMma0 + kMmaThreads;

// The MMA warpgroup's K loop over the ring: wgmma for stage i is committed, then stage i - 1 is known to have retired and
// its slot is handed back to the producers.  issue(i, s) queues the wgmmas of one stage.
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
__device__ __forceinline__ void mma_publish(const AccTile<BN> &acc, float *tile, uint64_t *tmem_full, int mt) {
    mma_group_sync();
    acc.store(tile, mt);
    mma_group_sync();
    if (mt == 0) mbar_arrive(tmem_full);
}

template <int BN, int STAGES>
struct SmemLayout {
    static constexpr int A_BYTES = BM * BK * 2;      // 16 KB
    static constexpr int B_BYTES = BN * BK * 2;
    static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
    static constexpr int BAR_OFF = STAGES * STAGE_BYTES;
    static constexpr int TOTAL = BAR_OFF + (2 * STAGES + 1) * 8 + 16 + 1024;   // + alignment slack
    static_assert(AccTile<BN>::BYTES <= BAR_OFF, "the accumulator tile is laid over the operand ring");
};

template <int BN, int STAGES, int A_MN, int B_MN>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_tcgen05_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, GemmArgs g) {
    using L = SmemLayout<BN, STAGES>;
    extern __shared__ unsigned char smem_raw[];
    unsigned char *smem = (unsigned char *)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);   // SW128 needs 1024 B
    uint64_t *full = (uint64_t *)(smem + L::BAR_OFF);
    uint64_t *empty = full + STAGES;
    uint64_t *tmem_full = empty + STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
    const int kb_total = (g.K + BK - 1) / BK;
    const int kb_lo = blockIdx.z * g.kblocks_per_split;
    const int kb_hi = min(kb_total, kb_lo + g.kblocks_per_split);
    const int nkb = kb_hi - kb_lo;

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        for (int s = 0; s < STAGES; ++s) { mbar_init(full + s, 1); mbar_init(empty + s, 1); }
        mbar_init(tmem_full, 1);
        fence_barrier_init();
    }
    __syncthreads();
    float *acc_tile = (float *)smem;

    if (warp == 0) {
        // ------------------------------------------------------------ TMA producer
        if (elect_one()) {
            for (int i = 0; i < nkb; ++i) {
                const int s = i % STAGES;
                const uint32_t ph = (i / STAGES) & 1;
                mbar_wait(empty + s, ph ^ 1);
                unsigned char *a_dst = smem + s * L::STAGE_BYTES;
                unsigned char *b_dst = a_dst + L::A_BYTES;
                mbar_expect_tx(full + s, L::STAGE_BYTES);
                const int k0 = (kb_lo + i) * BK;
                if (A_MN == 0) tma_load_2d(&tmA, full + s, a_dst, k0, m0);                 // box {64 k, 128 m}
                else {                                                                       // 2 boxes {64 m, 64 k}
                    tma_load_2d(&tmA, full + s, a_dst, m0, k0);
                    tma_load_2d(&tmA, full + s, a_dst + BK * 128, m0 + 64, k0);
                }
                if (B_MN == 0) tma_load_2d(&tmB, full + s, b_dst, k0, n0);                 // box {64 k, BN n}
                else {
#pragma unroll
                    for (int j = 0; j < BN / 64; ++j) tma_load_2d(&tmB, full + s, b_dst + j * BK * 128, n0 + 64 * j, k0);
                }
            }
        }
    } else if (threadIdx.x >= kGemmMma0) {
        // ------------------------------------------------------------ MMA warpgroup
        const int mt = threadIdx.x - kGemmMma0;
        AccTile<BN> acc;
        mma_ring(nkb, STAGES, full, empty, mt == 0, [&](int i, int s) {
            const uint32_t a_addr = smem_u32(smem + s * L::STAGE_BYTES);
            const uint32_t b_addr = a_addr + L::A_BYTES;
#pragma unroll
            for (int k = 0; k < BK / UMMA_K; ++k) {
                // K-major: 8-row groups 1024 B apart (SBO), advance 32 B per 16-deep step inside the 128 B atom; the
                //          tile's lower 64 rows start 64 * 128 B further on.
                // MN-major: 64-element M/N atoms BK*128 B apart (LBO), 8-row K groups 1024 B apart (SBO),
                //           advance 16 rows * 128 B per step; the lower 64 rows are the second atom.
                const uint64_t a_lo = A_MN == 0 ? make_desc(a_addr + k * 32, 16, 1024) : make_desc(a_addr + k * 2048, BK * 128, 1024);
                const uint64_t a_hi = A_MN == 0 ? make_desc(a_addr + 64 * 128 + k * 32, 16, 1024)
                                                : make_desc(a_addr + BK * 128 + k * 2048, BK * 128, 1024);
                const uint64_t bd = B_MN == 0 ? make_desc(b_addr + k * 32, 16, 1024) : make_desc(b_addr + k * 2048, BK * 128, 1024);
                acc.template mma<A_MN, B_MN>(a_lo, a_hi, bd, (i | k) != 0);
            }
        });
        if (nkb > 0) mma_publish<BN>(acc, acc_tile, tmem_full, mt);
    } else if (warp >= 2 && threadIdx.x < 192) {
        // ------------------------------------------------------------ epilogue (warps 2..5)
        epilogue_store<BN>(g, acc_tile, tmem_full, m0, n0, warp, lane, nkb > 0);
    }
}

// =====================================================================================================
// Implicit-GEMM convolution, stride 1, NHWC bf16  (backbones/crnn.py:46-49 nn.Conv2d; also its input gradient)
//
//   y[p, co] = sum_{tap, c} x[pixel(p) shifted by tap, c] * Wm[co, tap*C + c]          p = (n, ho, wo) flattened
//
// The im2col matrix never exists in HBM: warps 2..5 (one thread per output pixel of the 128-row tile) gather the
// 128-byte channel chunk of each row with zero-filling cp.async straight into the 128B-swizzled K-major smem tile
// that wgmma.mma_async reads (chunk j of row r lands at r*128 + ((j ^ (r & 7)) << 4)); the weight tile comes by TMA.
// The same kernel computes the input gradient: dgrad of a stride-1 convolution is a convolution of dz with the
// flipped / transposed weights and padding (k-1-p).  Requires C % 64 == 0.
// =====================================================================================================
struct ConvArgs {
    const bf16 *x;
    int N, H, W, C, kh, kw, ph, pw, Ho, Wo;
    int sh, sw, dh, dw;                 // stride and dilation (round 2: ResNet trunks; 1 / 1 for the CRNN layers)
    // TMA-A variant: the output space [N, Ho, Wo] is tiled by boxes of bw x bh x bn = 128 pixels; the width is cut
    // into segments of power-of-two widths (e.g. Wo = 65 -> one 64-wide segment + one 1-wide segment).
    struct Seg { int w0, bw, bh, bn, h_blocks, tile_begin; } seg[4];
    int nseg;
    GemmArgs g;        // M = N*Ho*Wo, N = Cout, K = kh*kw*C
};

__device__ __forceinline__ void tma_load_4d(const CUtensorMap *map, uint64_t *bar, void *dst, int c0, int c1, int c2, int c3) {
    asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
                 ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void cp_async16_zfill(uint32_t dst, const void *src, uint32_t src_bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}

// One 128-row tile per CTA: a second accumulator would double the MMA warpgroup's register need (BN registers per thread
// per tile), which is a limit of the one-warpgroup design, not a measured choice.
template <int BN, int STAGES>
struct ConvSmem {
    static constexpr int A_BYTES = BM * BK * 2;
    static constexpr int B_BYTES = BN * BK * 2;
    static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
    static constexpr int BAR_OFF = STAGES * STAGE_BYTES;
    static constexpr int TOTAL = BAR_OFF + (2 * STAGES + 1) * 8 + 16 + 1024;
};

// TMA_A = 1: "same"-padded convolutions whose 128-pixel tiles are whole row segments (W | 128 or 128 | W) fetch the
// activation tile with ONE 4-D TMA per K block (tap shift = signed coordinate offset, padding = TMA zero fill)
// instead of 1024 cp.async from the LSU.
template <int BN, int STAGES, int TMA_A>
__global__ void __launch_bounds__(kGemmThreads, 1)
conv_fprop_tcgen05_kernel(const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmX0,
                          const __grid_constant__ CUtensorMap tmX1, const __grid_constant__ CUtensorMap tmX2,
                          const __grid_constant__ CUtensorMap tmX3, ConvArgs a) {
    using L = ConvSmem<BN, STAGES>;
    static_assert(AccTile<BN>::BYTES <= L::BAR_OFF, "the accumulator tile is laid over the operand ring");
    extern __shared__ unsigned char smem_raw[];
    unsigned char *smem = (unsigned char *)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint64_t *full = (uint64_t *)(smem + L::BAR_OFF);
    uint64_t *empty = full + STAGES;
    uint64_t *tmem_full = empty + STAGES;
    const GemmArgs &g = a.g;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
    const int cchunks = a.C / BK;
    const int nkb = a.kh * a.kw * cchunks;

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&tmB);
        if (TMA_A) tma_prefetch_desc(&tmX0);
        for (int s = 0; s < STAGES; ++s) { mbar_init(full + s, TMA_A ? 1 : 1 + 128); mbar_init(empty + s, 1); }
        mbar_init(tmem_full, 1);
        fence_barrier_init();
    }
    __syncthreads();
    float *acc_tile = (float *)smem;

    if (warp == 0) {
        if (elect_one()) {                                   // weight tiles (and, with TMA_A, activation tiles) by TMA
            // TMA_A: this CTA owns tile blockIdx.x of the segment enumeration
            int tn = 0, th0 = 0, tw0 = 0;
            const CUtensorMap *tmX = &tmX0;
            if (TMA_A) {
                const int tile = (int)blockIdx.x;
                int sel = 0;
                for (int q = 1; q < a.nseg; ++q) if (tile >= a.seg[q].tile_begin) sel = q;
                const int lt = tile - a.seg[sel].tile_begin;
                const int nb = lt / a.seg[sel].h_blocks;
                tn = nb * a.seg[sel].bn;
                th0 = (lt - nb * a.seg[sel].h_blocks) * a.seg[sel].bh;
                tw0 = a.seg[sel].w0;
                tmX = sel == 0 ? &tmX0 : (sel == 1 ? &tmX1 : (sel == 2 ? &tmX2 : &tmX3));
            }
            int cc = 0, ti = 0, tj = 0;
            for (int i = 0; i < nkb; ++i) {
                const int s = i % STAGES;
                mbar_wait(empty + s, ((i / STAGES) & 1) ^ 1);
                mbar_expect_tx(full + s, TMA_A ? L::STAGE_BYTES : L::B_BYTES);
                if (TMA_A) {
                    tma_load_4d(tmX, full + s, smem + s * L::STAGE_BYTES, cc * BK, tw0 * a.sw + tj * a.dw - a.pw,
                                th0 * a.sh + ti * a.dh - a.ph, tn);
                    if (++cc == cchunks) { cc = 0; if (++tj == a.kw) { tj = 0; ++ti; } }
                }
                tma_load_2d(&tmB, full + s, smem + s * L::STAGE_BYTES + L::A_BYTES, i * BK, n0);
            }
        }
    } else if (threadIdx.x >= kGemmMma0) {
        // ------------------------------------------------------------ MMA warpgroup
        const int mt = threadIdx.x - kGemmMma0;
        AccTile<BN> acc;
        mma_ring(nkb, STAGES, full, empty, mt == 0, [&](int i, int s) {
            const uint32_t a_addr = smem_u32(smem + s * L::STAGE_BYTES);
            const uint32_t b_addr = a_addr + L::A_BYTES;
#pragma unroll
            for (int k = 0; k < BK / UMMA_K; ++k)
                acc.template mma<0, 0>(make_desc(a_addr + k * 32, 16, 1024), make_desc(a_addr + 64 * 128 + k * 32, 16, 1024),
                                       make_desc(b_addr + k * 32, 16, 1024), (i | k) != 0);
        });
        if (nkb > 0) mma_publish<BN>(acc, acc_tile, tmem_full, mt);
    } else if (warp < 2 || threadIdx.x >= 192) {
        // warp 1 and the padding warps have no role
    } else if (TMA_A) {
        const int tile = (int)blockIdx.x;
        int64_t prow = -1;
        int sel = 0;
        for (int q = 1; q < a.nseg; ++q) if (tile >= a.seg[q].tile_begin) sel = q;
        const int lt = tile - a.seg[sel].tile_begin;
        const int nb = lt / a.seg[sel].h_blocks;
        const int bw = a.seg[sel].bw, bh = a.seg[sel].bh;
        const int r = (warp & 3) * 32 + lane;                // tile row = (dn * bh + dh) * bw + dw
        const int dw = r % bw, dh = (r / bw) % bh, dn = r / (bw * bh);
        const int pn = nb * a.seg[sel].bn + dn, phh = (lt - nb * a.seg[sel].h_blocks) * bh + dh, pww = a.seg[sel].w0 + dw;
        if (pn < a.N && phh < a.Ho && pww < a.Wo) prow = ((int64_t)pn * a.Ho + phh) * a.Wo + pww;
        epilogue_store<BN>(g, acc_tile, tmem_full, 0, n0, warp, lane, nkb > 0, prow);
    } else {
        // ------------------------------------------------------------ activation gather (one thread = one tile row)
        const int r = threadIdx.x - 64;
        const int64_t p = (int64_t)m0 + r;
        const bool valid = p < g.M;
        int n = 0, ho = 0, wo = 0;
        if (valid) {
            wo = (int)(p % a.Wo);
            const int64_t t = p / a.Wo;
            ho = (int)(t % a.Ho);
            n = (int)(t / a.Ho);
        }
        const uint32_t row_off = (uint32_t)r * 128u;
        const uint32_t sw = (uint32_t)(r & 7);
        constexpr int D = STAGES >= 4 ? 3 : 2;                // cp.async groups in flight per thread
        static_assert(D - 1 < STAGES, "producer lookahead must be smaller than the ring");
        int cc = 0, ti = 0, tj = 0;
        for (int i = 0; i < nkb; ++i) {
            const int s = i % STAGES;
            mbar_wait(empty + s, ((i / STAGES) & 1) ^ 1);
            const int h = ho * a.sh + ti * a.dh - a.ph, w = wo * a.sw + tj * a.dw - a.pw;
            const bool ok = valid && h >= 0 && h < a.H && w >= 0 && w < a.W;
            const bf16 *src = ok ? a.x + ((((int64_t)n * a.H + h) * a.W + w) * a.C + cc * BK) : a.x;
            const uint32_t dst = smem_u32(smem + s * L::STAGE_BYTES) + row_off;
            const uint32_t nbytes = ok ? 16u : 0u;
#pragma unroll
            for (int j = 0; j < 8; ++j) cp_async16_zfill(dst + (((uint32_t)j ^ sw) << 4), src + j * 8, nbytes);
            cp_async_commit();
            if (i >= D - 1) {
                cp_async_wait<D - 1>();
                fence_proxy_async();                          // generic-proxy smem writes -> visible to wgmma
                mbar_arrive(full + (i - (D - 1)) % STAGES);
            }
            if (++cc == cchunks) { cc = 0; if (++tj == a.kw) { tj = 0; ++ti; } }
        }
        cp_async_wait<0>();
        fence_proxy_async();
        for (int i = (nkb >= D - 1 ? nkb - (D - 1) : 0); i < nkb; ++i) mbar_arrive(full + i % STAGES);
        epilogue_store<BN>(g, acc_tile, tmem_full, m0, n0, warp, lane, nkb > 0);
    }
}

// =====================================================================================================
// Implicit-GEMM weight gradient:  dW[co, tap*C + c] += sum_p dz[p, co] * x[pixel(p) shifted by tap, c]
// Both operands are MN-major and come by 4-D TMA: the reduction dimension (pixels) is tiled in row segments
// {RB w, 1 h, 1 n}; the tap shift is a signed coordinate offset and TMA zero-fills what falls outside the image, so
// padding needs no special case.  Split-K over the row segments, fp32 atomics into dW (pre-zeroed by the caller).
// =====================================================================================================
struct WgradArgs {
    int N, H, W, C, kh, kw, ph, pw, Ho, Wo, Cout;
    int sh, sw, dh, dw;
    int wboxes;                 // ceil(Wo / RB)
    int kb_total, kblocks_per_split;
    GemmArgs g;                 // M = Cout, N = kh*kw*C, C = dW, atomic = 1
};


template <int BN, int RB, int STAGES>
struct WgradSmem {
    static constexpr int A_BYTES = 2 * RB * 128;              // 128 output channels = 2 atoms of [RB rows][128 B]
    static constexpr int B_BYTES = (BN / 64) * RB * 128;
    static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
    static constexpr int BAR_OFF = STAGES * STAGE_BYTES;
    static constexpr int TOTAL = BAR_OFF + (2 * STAGES + 1) * 8 + 16 + 1024;
};

template <int BN, int RB, int STAGES>
__global__ void __launch_bounds__(kGemmThreads, 1)
conv_wgrad_tcgen05_kernel(const __grid_constant__ CUtensorMap tmDz, const __grid_constant__ CUtensorMap tmX, WgradArgs a) {
    using L = WgradSmem<BN, RB, STAGES>;
    static_assert(AccTile<BN>::BYTES <= L::BAR_OFF, "the accumulator tile is laid over the operand ring");
    extern __shared__ unsigned char smem_raw[];
    unsigned char *smem = (unsigned char *)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint64_t *full = (uint64_t *)(smem + L::BAR_OFF);
    uint64_t *empty = full + STAGES;
    uint64_t *tmem_full = empty + STAGES;
    const GemmArgs &g = a.g;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
    const int kb_lo = blockIdx.z * a.kblocks_per_split;
    const int kb_hi = min(a.kb_total, kb_lo + a.kblocks_per_split);
    const int nkb = kb_hi - kb_lo;

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&tmDz);
        tma_prefetch_desc(&tmX);
        for (int s = 0; s < STAGES; ++s) { mbar_init(full + s, 1); mbar_init(empty + s, 1); }
        mbar_init(tmem_full, 1);
        fence_barrier_init();
    }
    __syncthreads();
    float *acc_tile = (float *)smem;

    if (warp == 0) {
        if (elect_one()) {
            // the BN/64 column atoms of this tile: (tap, channel offset) each
            int at_i[BN / 64], at_j[BN / 64], at_c[BN / 64];
#pragma unroll
            for (int q = 0; q < BN / 64; ++q) {
                const int col = n0 + 64 * q;
                const int tap = col / a.C;
                at_c[q] = col - tap * a.C;
                at_i[q] = tap / a.kw;
                at_j[q] = tap - at_i[q] * a.kw;
            }
            for (int i = 0; i < nkb; ++i) {
                const int s = i % STAGES;
                mbar_wait(empty + s, ((i / STAGES) & 1) ^ 1);
                int kb = kb_lo + i;
                const int wb = kb % a.wboxes; kb /= a.wboxes;
                const int ho = kb % a.Ho;
                const int n = kb / a.Ho;
                unsigned char *a_dst = smem + s * L::STAGE_BYTES;
                unsigned char *b_dst = a_dst + L::A_BYTES;
                mbar_expect_tx(full + s, L::STAGE_BYTES);
                tma_load_4d(&tmDz, full + s, a_dst, m0, wb * RB, ho, n);
                tma_load_4d(&tmDz, full + s, a_dst + RB * 128, m0 + 64, wb * RB, ho, n);
#pragma unroll
                for (int q = 0; q < BN / 64; ++q) {
                    if (n0 + 64 * q < g.N)
                        tma_load_4d(&tmX, full + s, b_dst + q * RB * 128, at_c[q], wb * RB * a.sw + at_j[q] * a.dw - a.pw,
                                    ho * a.sh + at_i[q] * a.dh - a.ph, n);
                    else   // column atom beyond kh*kw*C: keep the transaction count with an all-out-of-bounds box
                        tma_load_4d(&tmX, full + s, b_dst + q * RB * 128, 0, -RB * a.sw - 8, 0, n);
                }
            }
        }
    } else if (threadIdx.x >= kGemmMma0) {
        // ------------------------------------------------------------ MMA warpgroup
        const int mt = threadIdx.x - kGemmMma0;
        AccTile<BN> acc;
        mma_ring(nkb, STAGES, full, empty, mt == 0, [&](int i, int s) {
            const uint32_t a_addr = smem_u32(smem + s * L::STAGE_BYTES);
            const uint32_t b_addr = a_addr + L::A_BYTES;
#pragma unroll
            for (int k = 0; k < RB / UMMA_K; ++k)
                acc.template mma<1, 1>(make_desc(a_addr + k * 2048, RB * 128, 1024), make_desc(a_addr + RB * 128 + k * 2048, RB * 128, 1024),
                                       make_desc(b_addr + k * 2048, RB * 128, 1024), (i | k) != 0);
        });
        if (nkb > 0) mma_publish<BN>(acc, acc_tile, tmem_full, mt);
    } else if (warp >= 2 && threadIdx.x < 192) {
        epilogue_store<BN>(g, acc_tile, tmem_full, m0, n0, warp, lane, nkb > 0);
    }
}

// =====================================================================================================
// Fused LSTM time step (decoders/crnn.py:13,17 nn.LSTM): recurrent GEMM + cell in ONE launch for both directions.
// Gate columns are stored UNIT-MAJOR (column 4*j + g holds gate g of hidden unit j; g = i,f,g,o) so that the 32
// accumulator columns a thread reads from the accumulator tile are 8 complete units.
//   forward : gates = Gx[t] + h_prev W_hh^T (+ bias);  c, h = cell(gates);  activated gates saved in place.
//   backward: dh = dY[t] + dG[t_next] W_hh ;  dG[t], dc = cell'(...)        (the GEMM feeds the cell directly)
// =====================================================================================================
struct LstmFwdDir {
    bf16 *gates;              // [B, 4H] unit-major: in = x-projection, out = activated gates
    const float *bias;        // [4H] unit-major, b_ih + b_hh
    const float *c_prev;      // [B, H] or NULL
    float *c_out;             // [B, H]
    bf16 *h_out;              // row stride ldh (slice of the [T, B, 2H] layer output)
    bf16 *h_next;             // [B, H] operand of the next step's GEMM
};
struct LstmFwdArgs { LstmFwdDir d[2]; int64_t ldh; int B, H, have_h; };

// Both LSTM step kernels: 64 output columns per CTA, a producer warp, 16 epilogue warps (4 row quarters x 4 groups of 16
// columns) and the MMA warpgroup: the cell arithmetic is transcendental-heavy and latency-bound, so it is spread over as
// many warps and CTAs as the tile shape allows.
constexpr int kLstmBN = 64;
constexpr int kLstmMma0 = 640;                      // 64 + 16 epilogue warps, padded to a warpgroup boundary
constexpr int kLstmThreads = kLstmMma0 + kMmaThreads;

template <int STAGES>
__global__ void __launch_bounds__(kLstmThreads, 1)
lstm_step_fwd_tcgen05_kernel(const __grid_constant__ CUtensorMap tmA0, const __grid_constant__ CUtensorMap tmA1,
                             const __grid_constant__ CUtensorMap tmB0, const __grid_constant__ CUtensorMap tmB1,
                             LstmFwdArgs a) {
    constexpr int BN = kLstmBN;
    using L = SmemLayout<BN, STAGES>;
    extern __shared__ unsigned char smem_raw[];
    unsigned char *smem = (unsigned char *)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint64_t *full = (uint64_t *)(smem + L::BAR_OFF);
    uint64_t *empty = full + STAGES;
    uint64_t *tmem_full = empty + STAGES;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int dir = blockIdx.z;
    const CUtensorMap *tmA = dir ? &tmA1 : &tmA0;
    const CUtensorMap *tmB = dir ? &tmB1 : &tmB0;
    const LstmFwdDir &q = a.d[dir];
    const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
    const int nkb = a.have_h ? a.H / BK : 0;

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(tmA);
        tma_prefetch_desc(tmB);
        for (int s = 0; s < STAGES; ++s) { mbar_init(full + s, 1); mbar_init(empty + s, 1); }
        mbar_init(tmem_full, 1);
        fence_barrier_init();
    }
    __syncthreads();
    float *acc_tile = (float *)smem;

    if (warp == 0) {
        if (elect_one()) {
            for (int i = 0; i < nkb; ++i) {
                const int s = i % STAGES;
                mbar_wait(empty + s, ((i / STAGES) & 1) ^ 1);
                mbar_expect_tx(full + s, L::STAGE_BYTES);
                tma_load_2d(tmA, full + s, smem + s * L::STAGE_BYTES, i * BK, m0);
                tma_load_2d(tmB, full + s, smem + s * L::STAGE_BYTES + L::A_BYTES, i * BK, n0);
            }
        }
    } else if (threadIdx.x >= kLstmMma0) {
        // ------------------------------------------------------------ MMA warpgroup
        const int mt = threadIdx.x - kLstmMma0;
        AccTile<BN> acc;
        mma_ring(nkb, STAGES, full, empty, mt == 0, [&](int i, int s) {
            const uint32_t a_addr = smem_u32(smem + s * L::STAGE_BYTES);
            const uint32_t b_addr = a_addr + L::A_BYTES;
#pragma unroll
            for (int k = 0; k < BK / UMMA_K; ++k)
                acc.template mma<0, 0>(make_desc(a_addr + k * 32, 16, 1024), make_desc(a_addr + 64 * 128 + k * 32, 16, 1024),
                                       make_desc(b_addr + k * 32, 16, 1024), (i | k) != 0);
        });
        if (nkb > 0) mma_publish<BN>(acc, acc_tile, tmem_full, mt);
    } else if (warp >= 2 && threadIdx.x < 64 + 16 * 32) {
        const int qd = warp & 3, grp = (warp - 2) >> 2;       // 32-row quarter of the tile, 16-column group
        const int row = m0 + qd * 32 + lane;
        if (nkb > 0) mbar_wait(tmem_full, 0);
        const int H = a.H;
        uint32_t r[16];
        if (nkb > 0) acc_ld<16>(acc_tile, AccTile<BN>::LD, qd * 32, grp * 16, r);
        else {
#pragma unroll
            for (int j = 0; j < 16; ++j) r[j] = 0;
        }
        const int col0 = n0 + grp * 16;                       // unit-major gate column: 4 hidden units
        if (row < a.B && col0 < 4 * H) {
            const int j0 = col0 >> 2;
            bf16 *gp = q.gates + (int64_t)row * 4 * H + col0;
            float pre[16];
#pragma unroll
            for (int v = 0; v < 2; ++v) {
                const uint4 pk = *reinterpret_cast<const uint4 *>(gp + v * 8);
                const __nv_bfloat162 *h2 = reinterpret_cast<const __nv_bfloat162 *>(&pk);
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const float2 f = __bfloat1622float2(h2[e]);
                    pre[v * 8 + 2 * e] = f.x;
                    pre[v * 8 + 2 * e + 1] = f.y;
                }
            }
            float bb[16];
#pragma unroll
            for (int v = 0; v < 4; ++v) {
                const float4 b4 = __ldg(reinterpret_cast<const float4 *>(q.bias + col0) + v);
                bb[4 * v] = b4.x; bb[4 * v + 1] = b4.y; bb[4 * v + 2] = b4.z; bb[4 * v + 3] = b4.w;
            }
            float cpv[4] = {0.f, 0.f, 0.f, 0.f};
            if (q.c_prev) {
                const float4 c4 = *reinterpret_cast<const float4 *>(q.c_prev + (int64_t)row * H + j0);
                cpv[0] = c4.x; cpv[1] = c4.y; cpv[2] = c4.z; cpv[3] = c4.w;
            }
            float act[16], cn[4], hn[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const float i_ = sigmoid_fast(pre[4 * u] + __uint_as_float(r[4 * u]) + bb[4 * u]);
                const float f_ = sigmoid_fast(pre[4 * u + 1] + __uint_as_float(r[4 * u + 1]) + bb[4 * u + 1]);
                const float g_ = tanh_fast(pre[4 * u + 2] + __uint_as_float(r[4 * u + 2]) + bb[4 * u + 2]);
                const float o_ = sigmoid_fast(pre[4 * u + 3] + __uint_as_float(r[4 * u + 3]) + bb[4 * u + 3]);
                cn[u] = f_ * cpv[u] + i_ * g_;
                hn[u] = o_ * tanh_fast(cn[u]);
                act[4 * u] = i_; act[4 * u + 1] = f_; act[4 * u + 2] = g_; act[4 * u + 3] = o_;
            }
#pragma unroll
            for (int v = 0; v < 2; ++v) {
                uint4 pk;
                __nv_bfloat162 *h2 = reinterpret_cast<__nv_bfloat162 *>(&pk);
#pragma unroll
                for (int e = 0; e < 4; ++e) h2[e] = __floats2bfloat162_rn(act[v * 8 + 2 * e], act[v * 8 + 2 * e + 1]);
                *reinterpret_cast<uint4 *>(gp + v * 8) = pk;
            }
            *reinterpret_cast<float4 *>(q.c_out + (int64_t)row * H + j0) = make_float4(cn[0], cn[1], cn[2], cn[3]);
            uint2 hp;
            __nv_bfloat162 *hh = reinterpret_cast<__nv_bfloat162 *>(&hp);
            hh[0] = __floats2bfloat162_rn(hn[0], hn[1]);
            hh[1] = __floats2bfloat162_rn(hn[2], hn[3]);
            *reinterpret_cast<uint2 *>(q.h_out + (int64_t)row * a.ldh + j0) = hp;
            *reinterpret_cast<uint2 *>(q.h_next + (int64_t)row * H + j0) = hp;
        }
    }
}

struct LstmBwdDir {
    const bf16 *gates;        // [B, 4H] activated gates of step t (unit-major)
    const float *c;           // [B, H] cell state of step t
    const float *c_prev;      // [B, H] or NULL
    const bf16 *dh_out;       // dY[t] slice, row stride ldh
    float *dc;                // [B, H] in/out
    bf16 *dgates;             // [B, 4H] unit-major, out
};
struct LstmBwdArgs { LstmBwdDir d[2]; int64_t ldh; int B, H, have_rec; };

template <int STAGES>
__global__ void __launch_bounds__(kLstmThreads, 1)
lstm_step_bwd_tcgen05_kernel(const __grid_constant__ CUtensorMap tmA0, const __grid_constant__ CUtensorMap tmA1,
                             const __grid_constant__ CUtensorMap tmB0, const __grid_constant__ CUtensorMap tmB1,
                             LstmBwdArgs a) {
    constexpr int BN = kLstmBN;     // 64 hidden units per CTA
    using L = SmemLayout<BN, STAGES>;
    extern __shared__ unsigned char smem_raw[];
    unsigned char *smem = (unsigned char *)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint64_t *full = (uint64_t *)(smem + L::BAR_OFF);
    uint64_t *empty = full + STAGES;
    uint64_t *tmem_full = empty + STAGES;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int dir = blockIdx.z;
    const CUtensorMap *tmA = dir ? &tmA1 : &tmA0;
    const CUtensorMap *tmB = dir ? &tmB1 : &tmB0;
    const LstmBwdDir &q = a.d[dir];
    const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
    const int nkb = a.have_rec ? (4 * a.H) / BK : 0;

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(tmA);
        tma_prefetch_desc(tmB);
        for (int s = 0; s < STAGES; ++s) { mbar_init(full + s, 1); mbar_init(empty + s, 1); }
        mbar_init(tmem_full, 1);
        fence_barrier_init();
    }
    __syncthreads();
    float *acc_tile = (float *)smem;

    if (warp == 0) {
        if (elect_one()) {
            for (int i = 0; i < nkb; ++i) {
                const int s = i % STAGES;
                mbar_wait(empty + s, ((i / STAGES) & 1) ^ 1);
                mbar_expect_tx(full + s, L::STAGE_BYTES);
                tma_load_2d(tmA, full + s, smem + s * L::STAGE_BYTES, i * BK, m0);          // dG_next [B, 4H], K-major
                tma_load_2d(tmB, full + s, smem + s * L::STAGE_BYTES + L::A_BYTES, n0, i * BK);   // W_hh [4H, H], MN-major
            }
        }
    } else if (threadIdx.x >= kLstmMma0) {
        // ------------------------------------------------------------ MMA warpgroup
        const int mt = threadIdx.x - kLstmMma0;
        AccTile<BN> acc;
        mma_ring(nkb, STAGES, full, empty, mt == 0, [&](int i, int s) {
            const uint32_t a_addr = smem_u32(smem + s * L::STAGE_BYTES);
            const uint32_t b_addr = a_addr + L::A_BYTES;
#pragma unroll
            for (int k = 0; k < BK / UMMA_K; ++k)
                acc.template mma<0, 1>(make_desc(a_addr + k * 32, 16, 1024), make_desc(a_addr + 64 * 128 + k * 32, 16, 1024),
                                       make_desc(b_addr + k * 2048, BK * 128, 1024), (i | k) != 0);
        });
        if (nkb > 0) mma_publish<BN>(acc, acc_tile, tmem_full, mt);
    } else if (warp >= 2 && threadIdx.x < 64 + 16 * 32) {
        const int qd = warp & 3, grp = (warp - 2) >> 2;
        const int row = m0 + qd * 32 + lane;
        if (nkb > 0) mbar_wait(tmem_full, 0);
        const int H = a.H;
        uint32_t r[16];
        if (nkb > 0) acc_ld<16>(acc_tile, AccTile<BN>::LD, qd * 32, grp * 16, r);
        else {
#pragma unroll
            for (int j = 0; j < 16; ++j) r[j] = 0;
        }
        const int j0 = n0 + grp * 16;                          // first of 16 hidden units
        if (row < a.B && j0 < H) {
            const bf16 *gp = q.gates + (int64_t)row * 4 * H + 4 * j0;
            const bf16 *dyp = q.dh_out + (int64_t)row * a.ldh + j0;
            const float *cp = q.c + (int64_t)row * H + j0;
            const float *cpp = q.c_prev ? q.c_prev + (int64_t)row * H + j0 : nullptr;
            float *dcp = q.dc + (int64_t)row * H + j0;
            bf16 *dgp = q.dgates + (int64_t)row * 4 * H + 4 * j0;
#pragma unroll
            for (int v = 0; v < 2; ++v) {                      // 8 units per 16-byte vector of dY
                const uint4 dyk = *reinterpret_cast<const uint4 *>(dyp + v * 8);
                const __nv_bfloat162 *dy2 = reinterpret_cast<const __nv_bfloat162 *>(&dyk);
                float dyf[8], cf[8], cpf[8], dcf[8];
#pragma unroll
                for (int e = 0; e < 4; ++e) { const float2 f = __bfloat1622float2(dy2[e]); dyf[2 * e] = f.x; dyf[2 * e + 1] = f.y; }
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const float4 c4 = *reinterpret_cast<const float4 *>(cp + v * 8 + 4 * e);
                    cf[4 * e] = c4.x; cf[4 * e + 1] = c4.y; cf[4 * e + 2] = c4.z; cf[4 * e + 3] = c4.w;
                    const float4 d4 = *reinterpret_cast<const float4 *>(dcp + v * 8 + 4 * e);
                    dcf[4 * e] = d4.x; dcf[4 * e + 1] = d4.y; dcf[4 * e + 2] = d4.z; dcf[4 * e + 3] = d4.w;
                    float4 p4 = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (cpp) p4 = *reinterpret_cast<const float4 *>(cpp + v * 8 + 4 * e);
                    cpf[4 * e] = p4.x; cpf[4 * e + 1] = p4.y; cpf[4 * e + 2] = p4.z; cpf[4 * e + 3] = p4.w;
                }
                float dgf[32];
#pragma unroll
                for (int h = 0; h < 4; ++h) {                  // 2 units (8 gate values) per 16-byte vector of gates
                    const uint4 gk = *reinterpret_cast<const uint4 *>(gp + v * 32 + h * 8);
                    const __nv_bfloat162 *g2 = reinterpret_cast<const __nv_bfloat162 *>(&gk);
#pragma unroll
                    for (int w2 = 0; w2 < 2; ++w2) {
                        const int uu = h * 2 + w2;             // unit inside this group of 8
                        const float2 fi = __bfloat1622float2(g2[2 * w2]);       // (i, f)
                        const float2 fg = __bfloat1622float2(g2[2 * w2 + 1]);   // (g, o)
                        const float i_ = fi.x, f_ = fi.y, g_ = fg.x, o_ = fg.y;
                        const float dh = dyf[uu] + __uint_as_float(r[v * 8 + uu]);
                        const float tc = tanh_fast(cf[uu]);
                        const float dct = dcf[uu] + dh * o_ * (1.f - tc * tc);
                        dgf[uu * 4] = dct * g_ * i_ * (1.f - i_);
                        dgf[uu * 4 + 1] = dct * cpf[uu] * f_ * (1.f - f_);
                        dgf[uu * 4 + 2] = dct * i_ * (1.f - g_ * g_);
                        dgf[uu * 4 + 3] = dh * tc * o_ * (1.f - o_);
                        dcf[uu] = dct * f_;
                    }
                }
#pragma unroll
                for (int e = 0; e < 2; ++e)
                    *reinterpret_cast<float4 *>(dcp + v * 8 + 4 * e) = make_float4(dcf[4 * e], dcf[4 * e + 1], dcf[4 * e + 2], dcf[4 * e + 3]);
#pragma unroll
                for (int h = 0; h < 4; ++h) {
                    uint4 pk;
                    __nv_bfloat162 *p2 = reinterpret_cast<__nv_bfloat162 *>(&pk);
#pragma unroll
                    for (int e = 0; e < 4; ++e) p2[e] = __floats2bfloat162_rn(dgf[h * 8 + 2 * e], dgf[h * 8 + 2 * e + 1]);
                    *reinterpret_cast<uint4 *>(dgp + v * 32 + h * 8) = pk;
                }
            }
        }
    }
}

template <int BN, int STAGES, int A_MN, int B_MN>
int launch(const CUtensorMap &ta, const CUtensorMap &tb, const GemmArgs &g, int splits, cudaStream_t st) {
    using L = SmemLayout<BN, STAGES>;
    auto kern = gemm_tcgen05_kernel<BN, STAGES, A_MN, B_MN>;
    { int rc_attr = ensure_dyn_smem((const void *)kern, L::TOTAL, "gemm_tcgen05 smem attr"); if (rc_attr) return rc_attr; }
    dim3 grid((unsigned)ceil_div(g.M, BM), (unsigned)ceil_div(g.N, BN), (unsigned)splits);
    kern<<<grid, kGemmThreads, L::TOTAL, st>>>(ta, tb, g);
    return check_launch("gemm_tcgen05_kernel");
}

// 4-D bf16 NHWC tensor map {C, W, H, N}, box {64, box_w, 1, 1}
// sw / sh > 1: strided traversal (every sw-th column, sh-th row) -- the box then spans box_w * sw columns of the tensor and
// delivers box_w of them (cuTensorMapEncodeTiled elementStrides)
int make_map_nhwc(CUtensorMap *m, const void *base, int64_t C, int64_t W, int64_t H, int64_t N, int box_w, int box_h = 1,
                  int box_n = 1, int sw = 1, int sh = 1) {
    EncodeTiledFn fn = encode_fn();
    if (!fn) { set_cuda_error(cudaErrorUnknown, "cuTensorMapEncodeTiled entry point"); return MR_ERR_CUDA; }
    cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
    cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
    cuuint32_t box[4] = {64, (cuuint32_t)(box_w * sw), (cuuint32_t)(box_h * sh), (cuuint32_t)box_n};
    cuuint32_t estr[4] = {1, (cuuint32_t)sw, (cuuint32_t)sh, 1};
    if (box[1] > 256 || box[2] > 256) { set_cuda_error(cudaErrorInvalidValue, "conv tensor map: strided box too large"); return MR_ERR_UNSUPPORTED; }
    CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void *>(base), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_cuda_error(cudaErrorInvalidValue, "cuTensorMapEncodeTiled(4d)"); return MR_ERR_CUDA; }
    return MR_OK;
}

template <int BN, int STAGES, int TMA_A>
int launch_conv(const CUtensorMap &tb, const CUtensorMap *tx, const ConvArgs &a, int tiles, cudaStream_t st) {
    using L = ConvSmem<BN, STAGES>;
    auto kern = conv_fprop_tcgen05_kernel<BN, STAGES, TMA_A>;
    { int rc_attr = ensure_dyn_smem((const void *)kern, L::TOTAL, "conv_fprop smem attr"); if (rc_attr) return rc_attr; }
    dim3 grid(TMA_A ? (unsigned)tiles : (unsigned)ceil_div(a.g.M, BM), (unsigned)ceil_div(a.g.N, BN), 1);
    kern<<<grid, kGemmThreads, L::TOTAL, st>>>(tb, tx[0], tx[1], tx[2], tx[3], a);
    return check_launch("conv_fprop_tcgen05_kernel");
}

template <int BN, int RB, int STAGES>
int launch_wgrad(const CUtensorMap &tdz, const CUtensorMap &tx, const WgradArgs &a, int splits, cudaStream_t st) {
    using L = WgradSmem<BN, RB, STAGES>;
    auto kern = conv_wgrad_tcgen05_kernel<BN, RB, STAGES>;
    { int rc_attr = ensure_dyn_smem((const void *)kern, L::TOTAL, "conv_wgrad smem attr"); if (rc_attr) return rc_attr; }
    dim3 grid((unsigned)ceil_div(a.g.M, BM), (unsigned)ceil_div(a.g.N, BN), (unsigned)splits);
    kern<<<grid, kGemmThreads, L::TOTAL, st>>>(tdz, tx, a);
    return check_launch("conv_wgrad_tcgen05_kernel");
}

}  // namespace

extern "C" {

/* bf16 GEMM on wgmma/TMA.  transA = 0: A stored [M,K] (lda >= K); transA = 1: A stored [K,M] (lda >= M).
 * transB = 1: B stored [N,K] (ldb >= K);  transB = 0: B stored [K,N] (ldb >= N).   [same convention as mr_gemm]
 * Supported operand forms: (transA, transB) = (0, 1) "NT", (0, 0) "NN" and (1, 0) "TN".  lda, ldb multiples of 8, bases 16-byte
 * aligned.  out_dtype 0 = fp32, 1 = bf16.  beta must be 0 or 1; beta = 1 (fp32 only) accumulates atomically and allows
 * split-K (splits > 1).  Returns MR_ERR_UNSUPPORTED for anything else so that the caller can route to mr_gemm. */
int mr_gemm_tcgen05(const void *A, const void *B, void *C, int64_t M, int64_t N, int64_t K, int64_t lda, int64_t ldb,
                    int64_t ldc, int transA, int transB, int out_dtype, const float *bias, int relu, float beta,
                    int splits, void *stream) {
    if (M < 0 || N < 0 || K < 0) return MR_ERR_BAD_SHAPE;
    if (M == 0 || N == 0) return MR_OK;
    if (!A || !B || !C) return MR_ERR_NULL_POINTER;
    const bool nt = (transA == 0 && transB == 1), tn = (transA == 1 && transB == 0), nn = (transA == 0 && transB == 0);
    if (!nt && !tn && !nn) return MR_ERR_UNSUPPORTED;
    if (lda % 8 || ldb % 8 || ((uintptr_t)A % 16) || ((uintptr_t)B % 16)) return MR_ERR_UNSUPPORTED;
    if (beta != 0.f && (beta != 1.f || out_dtype != 0)) return MR_ERR_UNSUPPORTED;
    if (K == 0 || M > (1LL << 31) - 256 || N > (1LL << 31) - 256 || K > (1LL << 31) - 256) return MR_ERR_UNSUPPORTED;
    if (splits < 1) splits = 1;
    if (splits > 1 && beta != 1.f) return MR_ERR_UNSUPPORTED;
    cudaStream_t st = (cudaStream_t)stream;
    const int BN = N > 64 ? 128 : 64;
    CUtensorMap ta, tb;
    int rc;
    if (nt) {
        rc = make_map(&ta, A, K, M, lda, BK, BM);
        if (rc) return rc;
        rc = make_map(&tb, B, K, N, ldb, BK, BN);
    } else if (nn) {
        rc = make_map(&ta, A, K, M, lda, BK, BM);
        if (rc) return rc;
        rc = make_map(&tb, B, N, K, ldb, 64, BK);
    } else {
        rc = make_map(&ta, A, M, K, lda, 64, BK);
        if (rc) return rc;
        rc = make_map(&tb, B, N, K, ldb, 64, BK);
    }
    if (rc) return rc;
    GemmArgs g;
    g.M = (int)M; g.N = (int)N; g.K = (int)K; g.ldc = ldc; g.C = C; g.bias = bias; g.relu = relu;
    g.out_bf16 = out_dtype == 1; g.atomic = beta == 1.f;
    const int kb_total = (int)ceil_div(K, BK);
    if (splits > kb_total) splits = kb_total;
    g.kblocks_per_split = (int)ceil_div(kb_total, splits);
    splits = (int)ceil_div(kb_total, g.kblocks_per_split);
#define MR_LAUNCH(BNV, STV)                                                              \
    (nt ? launch<BNV, STV, 0, 0>(ta, tb, g, splits, st)                                  \
        : (nn ? launch<BNV, STV, 0, 1>(ta, tb, g, splits, st) : launch<BNV, STV, 1, 1>(ta, tb, g, splits, st)))
    if (BN == 128) return MR_LAUNCH(128, 6);
    return MR_LAUNCH(64, 8);
#undef MR_LAUNCH
}

/* Implicit-GEMM stride-1 convolution on NHWC bf16:  y[N*Ho*Wo, Cout] = conv(x[N,H,W,C], Wm[Cout, kh*kw*C]) (+bias, ReLU).
 * C % 64 == 0, Wm row pitch = kh*kw*C.  With flipped/transposed weights and padding (k-1-p) it is the input gradient. */
int mr_conv_fprop_tcgen05(const void *x, const void *Wm, void *y, int N, int H, int W, int C, int Cout, int kh, int kw,
                          int ph, int pw, int out_dtype, const float *bias, int relu, void *stream) {
    return mr_conv2d_fprop_tcgen05(x, Wm, y, N, H, W, C, Cout, kh, kw, 1, 1, ph, pw, 1, 1, out_dtype, bias, relu, stream);
}

/* General form: stride (sh, sw) and dilation (dh, dw) -- nn.Conv2d of the ResNet / PPM / FPN trunks (backbones/resnet.py:110-256,
 * resnet_dilated.py:50-69).  The tap shift is a TMA coordinate offset scaled by the dilation; a stride is the tensor map's
 * traversal stride (every s-th column / row of the box is delivered), so the kernel itself is unchanged. */
int mr_conv2d_fprop_tcgen05(const void *x, const void *Wm, void *y, int N, int H, int W, int C, int Cout, int kh, int kw,
                            int sh, int sw, int ph, int pw, int dh, int dw, int out_dtype, const float *bias, int relu,
                            void *stream) {
    if (N < 0 || H <= 0 || W <= 0 || C <= 0 || Cout <= 0 || kh <= 0 || kw <= 0 || ph < 0 || pw < 0 || sh <= 0 || sw <= 0 ||
        dh <= 0 || dw <= 0) return MR_ERR_BAD_SHAPE;
    if (N == 0) return MR_OK;
    if (!x || !Wm || !y) return MR_ERR_NULL_POINTER;
    if (C % 64 || ((uintptr_t)x % 16) || ((uintptr_t)Wm % 16)) return MR_ERR_UNSUPPORTED;
    ConvArgs a;
    a.x = (const bf16 *)x; a.N = N; a.H = H; a.W = W; a.C = C; a.kh = kh; a.kw = kw; a.ph = ph; a.pw = pw;
    a.sh = sh; a.sw = sw; a.dh = dh; a.dw = dw;
    a.Ho = (H + 2 * ph - dh * (kh - 1) - 1) / sh + 1; a.Wo = (W + 2 * pw - dw * (kw - 1) - 1) / sw + 1;
    if (a.Ho <= 0 || a.Wo <= 0 || H + 2 * ph < dh * (kh - 1) + 1 || W + 2 * pw < dw * (kw - 1) + 1) return MR_ERR_BAD_SHAPE;
    const int64_t P = (int64_t)N * a.Ho * a.Wo, K = (int64_t)kh * kw * C;
    if (P > (1LL << 31) - 256) return MR_ERR_UNSUPPORTED;
    a.g.M = (int)P; a.g.N = Cout; a.g.K = (int)K; a.g.ldc = Cout; a.g.C = y; a.g.bias = bias; a.g.relu = relu;
    a.g.out_bf16 = out_dtype == 1; a.g.atomic = 0; a.g.kblocks_per_split = 0;
    const int BN = Cout > 64 ? 128 : 64;
    CUtensorMap tb;
    int rc = make_map(&tb, Wm, K, Cout, K, BK, BN);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    /* TMA-A variant: tile the output space with boxes of 128 pixels, width cut into power-of-two segments. */
    static const bool no_tma_a = getenv("MR_CONV_NO_TMA_A") != nullptr;
    a.nseg = 0;
    CUtensorMap tx[4];
    int tiles = 0;
    if (!no_tma_a) {
        int w0 = 0;
        bool ok = true;
        while (w0 < a.Wo) {
            if (a.nseg == 4) { ok = false; break; }
            int bw = 128;
            while (bw > a.Wo - w0) bw >>= 1;
            int nrep = (a.Wo - w0) / bw;                  /* consecutive segments of this width share geometry */
            int bh = 1;
            while (bh * 2 <= a.Ho && bw * bh * 2 <= 128) bh <<= 1;
            const int bn = 128 / (bw * bh);
            const int h_blocks = (int)ceil_div(a.Ho, bh), n_blocks = (int)ceil_div(N, bn);
            for (int rep = 0; rep < nrep && ok; ++rep) {
                if (a.nseg == 4) { ok = false; break; }
                ConvArgs::Seg &sg = a.seg[a.nseg];
                sg.w0 = w0; sg.bw = bw; sg.bh = bh; sg.bn = bn; sg.h_blocks = h_blocks; sg.tile_begin = tiles;
                rc = make_map_nhwc(&tx[a.nseg], x, C, W, H, N, bw, bh, bn, sw, sh);
                if (rc == MR_ERR_UNSUPPORTED) { ok = false; break; }
                if (rc) return rc;
                tiles += h_blocks * n_blocks;
                ++a.nseg;
                w0 += bw;
            }
        }
        if (ok && a.nseg > 0) {
            for (int q = a.nseg; q < 4; ++q) tx[q] = tx[0];
            /* shallow rings leave room for 2-3 CTAs per SM, so one CTA's epilogue overlaps another's main loop
             * (the kernel is not persistent); MR_CONV_SHALLOW=0/1 overrides the default for experiments. */
            static const char *sh_env = getenv("MR_CONV_SHALLOW");
            const bool shallow = sh_env ? sh_env[0] == '1' : true;
            if (shallow) {
                if (BN == 128) return launch_conv<128, 3, 1>(tb, tx, a, tiles, st);
                return launch_conv<64, 3, 1>(tb, tx, a, tiles, st);
            }
            if (BN == 128) return launch_conv<128, 6, 1>(tb, tx, a, tiles, st);
            return launch_conv<64, 8, 1>(tb, tx, a, tiles, st);
        }
        a.nseg = 0;
    }
    for (int q = 0; q < 4; ++q) tx[q] = tb;
    if (BN == 128) return launch_conv<128, 6, 0>(tb, tx, a, 0, st);
    return launch_conv<64, 8, 0>(tb, tx, a, 0, st);
}

/* Implicit-GEMM weight gradient: dWm[Cout, kh*kw*C] (fp32, ACCUMULATED atomically: zero it first) from
 * dz[N,Ho,Wo,Cout] and x[N,H,W,C] (NHWC bf16, stride-1 geometry).  C % 64 == 0 and Cout % 8 == 0. */
int mr_conv_wgrad_tcgen05(const void *dz, const void *x, float *dWm, int N, int H, int W, int C, int Cout, int kh, int kw,
                          int ph, int pw, int splits, void *stream) {
    return mr_conv2d_wgrad_tcgen05(dz, x, dWm, N, H, W, C, Cout, kh, kw, 1, 1, ph, pw, 1, 1, splits, stream);
}

int mr_conv2d_wgrad_tcgen05(const void *dz, const void *x, float *dWm, int N, int H, int W, int C, int Cout, int kh, int kw,
                            int sh, int sw, int ph, int pw, int dh, int dw, int splits, void *stream) {
    if (N < 0 || H <= 0 || W <= 0 || C <= 0 || Cout <= 0 || kh <= 0 || kw <= 0 || ph < 0 || pw < 0 || sh <= 0 || sw <= 0 ||
        dh <= 0 || dw <= 0) return MR_ERR_BAD_SHAPE;
    if (N == 0) return MR_OK;
    if (!dz || !x || !dWm) return MR_ERR_NULL_POINTER;
    if (C % 64 || Cout % 8 || ((uintptr_t)x % 16) || ((uintptr_t)dz % 16)) return MR_ERR_UNSUPPORTED;
    WgradArgs a;
    a.N = N; a.H = H; a.W = W; a.C = C; a.kh = kh; a.kw = kw; a.ph = ph; a.pw = pw; a.Cout = Cout;
    a.sh = sh; a.sw = sw; a.dh = dh; a.dw = dw;
    a.Ho = (H + 2 * ph - dh * (kh - 1) - 1) / sh + 1; a.Wo = (W + 2 * pw - dw * (kw - 1) - 1) / sw + 1;
    if (a.Ho <= 0 || a.Wo <= 0 || H + 2 * ph < dh * (kh - 1) + 1 || W + 2 * pw < dw * (kw - 1) + 1) return MR_ERR_BAD_SHAPE;
    const int K = kh * kw * C;
    const bool rb80 = (a.Wo > 64 && a.Wo <= 80);
    const int RB = rb80 ? 80 : 64;
    a.wboxes = (int)ceil_div(a.Wo, RB);
    a.kb_total = N * a.Ho * a.wboxes;
    if (splits < 1) splits = 1;
    if (splits > a.kb_total) splits = a.kb_total;
    a.kblocks_per_split = (int)ceil_div(a.kb_total, splits);
    splits = (int)ceil_div(a.kb_total, a.kblocks_per_split);
    a.g.M = Cout; a.g.N = K; a.g.K = 0; a.g.ldc = K; a.g.C = dWm; a.g.bias = nullptr; a.g.relu = 0; a.g.out_bf16 = 0;
    a.g.atomic = 1; a.g.kblocks_per_split = a.kblocks_per_split;
    CUtensorMap tdz, tx;
    int rc = make_map_nhwc(&tdz, dz, Cout, a.Wo, a.Ho, N, RB);
    if (rc) return rc;
    rc = make_map_nhwc(&tx, x, C, W, H, N, RB, 1, 1, sw, 1);      /* rows are addressed one at a time: only the width strides */
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const int BN = K > 64 ? 128 : 64;
    if (rb80) {
        if (BN == 128) return launch_wgrad<128, 80, 4>(tdz, tx, a, splits, st);
        return launch_wgrad<64, 80, 6>(tdz, tx, a, splits, st);
    }
    if (BN == 128) return launch_wgrad<128, 64, 6>(tdz, tx, a, splits, st);
    return launch_wgrad<64, 64, 8>(tdz, tx, a, splits, st);
}

/* Fused LSTM steps (both directions per launch).  Unit-major gate layout (column 4*j + g).  H % 64 == 0.
 * h_prev[d]: [B,H] bf16 operand of this step's recurrent GEMM (ignored when have_h == 0, i.e. the first step);
 * Whh[d]: [4H, H] bf16 unit-major rows.  Per-direction pointer arguments are HOST arrays of 2 device pointers. */
int mr_lstm_step_fwd_tcgen05(const void *const *h_prev, const void *const *Whh, void *const *gates,
                             const float *const *bias, const float *const *c_prev, float *const *c_out,
                             void *const *h_out, int64_t ldh, void *const *h_next, int have_h, int B, int H,
                             void *stream) {
    if (B <= 0 || H <= 0 || H % 64) return MR_ERR_UNSUPPORTED;
    LstmFwdArgs a;
    a.ldh = ldh; a.B = B; a.H = H; a.have_h = have_h;
    CUtensorMap ta[2], tb[2];
    for (int d = 0; d < 2; ++d) {
        if (!h_prev[d] || !Whh[d] || !gates[d] || !bias[d] || !c_out[d] || !h_out[d] || !h_next[d]) return MR_ERR_NULL_POINTER;
        int rc = make_map(&ta[d], h_prev[d], H, B, H, BK, BM);
        if (rc) return rc;
        rc = make_map(&tb[d], Whh[d], H, 4 * H, H, BK, kLstmBN);
        if (rc) return rc;
        a.d[d].gates = (bf16 *)gates[d]; a.d[d].bias = bias[d]; a.d[d].c_prev = c_prev[d]; a.d[d].c_out = c_out[d];
        a.d[d].h_out = (bf16 *)h_out[d]; a.d[d].h_next = (bf16 *)h_next[d];
    }
    using L = SmemLayout<kLstmBN, 4>;
    auto kern = lstm_step_fwd_tcgen05_kernel<4>;
    { int rc_attr = ensure_dyn_smem((const void *)kern, L::TOTAL, "lstm fwd smem attr"); if (rc_attr) return rc_attr; }
    dim3 grid((unsigned)ceil_div(B, BM), (unsigned)(4 * H / kLstmBN), 2);
    kern<<<grid, kLstmThreads, L::TOTAL, (cudaStream_t)stream>>>(ta[0], ta[1], tb[0], tb[1], a);
    return check_launch("lstm_step_fwd_tcgen05_kernel");
}

/* dG_next[d]: [B,4H] bf16 gate gradients of the step processed before this one (ignored when have_rec == 0). */
int mr_lstm_step_bwd_tcgen05(const void *const *dG_next, const void *const *Whh, const void *const *gates,
                             const float *const *c, const float *const *c_prev, const void *const *dh_out, int64_t ldh,
                             float *const *dc, void *const *dgates, int have_rec, int B, int H, void *stream) {
    if (B <= 0 || H <= 0 || H % 64) return MR_ERR_UNSUPPORTED;
    LstmBwdArgs a;
    a.ldh = ldh; a.B = B; a.H = H; a.have_rec = have_rec;
    CUtensorMap ta[2], tb[2];
    for (int d = 0; d < 2; ++d) {
        if (!dG_next[d] || !Whh[d] || !gates[d] || !c[d] || !dh_out[d] || !dc[d] || !dgates[d]) return MR_ERR_NULL_POINTER;
        int rc = make_map(&ta[d], dG_next[d], 4 * H, B, 4 * H, BK, BM);
        if (rc) return rc;
        rc = make_map(&tb[d], Whh[d], H, 4 * H, H, 64, BK);
        if (rc) return rc;
        a.d[d].gates = (const bf16 *)gates[d]; a.d[d].c = c[d]; a.d[d].c_prev = c_prev[d];
        a.d[d].dh_out = (const bf16 *)dh_out[d]; a.d[d].dc = dc[d]; a.d[d].dgates = (bf16 *)dgates[d];
    }
    using L = SmemLayout<kLstmBN, 6>;
    auto kern = lstm_step_bwd_tcgen05_kernel<6>;
    { int rc_attr = ensure_dyn_smem((const void *)kern, L::TOTAL, "lstm bwd smem attr"); if (rc_attr) return rc_attr; }
    dim3 grid((unsigned)ceil_div(B, BM), (unsigned)(H / kLstmBN), 2);
    kern<<<grid, kLstmThreads, L::TOTAL, (cudaStream_t)stream>>>(ta[0], ta[1], tb[0], tb[1], a);
    return check_launch("lstm_step_bwd_tcgen05_kernel");
}

}  // extern "C"
