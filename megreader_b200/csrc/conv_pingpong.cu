// Persistent ping-pong implicit-GEMM convolution, stride 1, NHWC bf16 -> bf16: the convolutions of the CRNN backbone
// (backbones/crnn.py:46-49 nn.Conv2d) and their input gradients.
//
//   y[p, co] = sum_{tap, c} x[pixel(p) shifted by tap, c] * Wm[co, tap*C + c]          p = (n, ho, wo) flattened
//
// Warp roles (384 threads, one CTA per SM, grid = min(tiles, SMs)):
//   warpgroup 0      producer: gives up registers (setmaxnreg 40); one elected lane streams the (activation, weight)
//                    K blocks of every tile this CTA owns through ONE ring of STAGES stages.  The ring position and the
//                    mbarrier phases run on across tiles, so no tile starts from an empty ring.
//   warpgroups 1, 2  consumers (setmaxnreg 232): each owns a whole 128 x BN output tile with its fp32 accumulator in
//                    registers.  They take the CTA's tiles in turn, and an order barrier alternates their main loops, so
//                    one consumer's epilogue (fragments -> bf16 -> stmatrix -> TMA store) runs while the other one keeps
//                    the tensor cores busy.
// Tiles are handed out statically, strided by gridDim.x; the Cout tiles of one 128-pixel tile are adjacent in that order,
// so they run on neighbouring CTAs at the same time and the activation box is read from HBM once and then hit in L2.
//
// The activation tile is the 4-D TMA box of plan_conv_segments (wgmma.cuh), exactly as conv_fprop_tcgen05_kernel<*,*,1>
// loads it: the tap shift is a signed coordinate offset and padding is TMA zero fill.  The output tile is stored with a
// box of the same geometry over y, so the segmented tiles of Wo = 65 need no index arithmetic and TMA clips what falls
// outside the tensor.  K order (tap-major 64-channel blocks) and instruction shape (two m64nBNk16 per 16-deep step) are those
// of conv_fprop_tcgen05_kernel, so every output element is the same fp32 sum rounded the same way: the results are
// bit-identical.
#include "wgmma.cuh"
#include <algorithm>

namespace {

constexpr int kPpThreads = 384;
constexpr int kPpProducerRegs = 40;
constexpr int kPpConsumerRegs = 232;       // 128 * 40 + 256 * 232 <= 65536
static_assert(128 * kPpProducerRegs + 256 * kPpConsumerRegs <= 65536, "register file");

// Named barriers (0 is __syncthreads): the consumers' turn barriers, and one per consumer for its epilogue.
constexpr int kBarTurn0 = 1, kBarTurn1 = 2, kBarEpi0 = 3;

// STAGES x (A 128x64, B BNx64) from a 1024-byte aligned base, then one bf16 output tile per consumer (BN/64 slices of
// 128 rows x 128 B, the TMA store boxes), then the barriers full[STAGES], empty[STAGES].
template <int BN> struct PpSmem {
    static constexpr int STAGES = BN == 128 ? 5 : 8;
    static constexpr int A_BYTES = BM * BK * 2;
    static constexpr int B_BYTES = BN * BK * 2;
    static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
    static constexpr int SLICE_BYTES = BM * 64 * 2;
    static constexpr int OUT_BYTES = (BN / 64) * SLICE_BYTES;
    static constexpr int OUT_OFF = STAGES * STAGE_BYTES;
    static constexpr int BAR_OFF = OUT_OFF + 2 * OUT_BYTES;
    static constexpr int TOTAL = BAR_OFF + 2 * STAGES * 8 + 1024;   // + alignment slack
    static_assert(TOTAL <= 232448, "227 KB of opt-in shared memory");
};

struct PpConvArgs {
    int C, Cout, kh, kw, ph, pw;
    int cout_tiles, tiles;            // tiles = 128-pixel tiles x cout_tiles
    int nseg;
    ConvSeg seg[kMaxConvSegs];
};

struct PixTile { int n, h0, w0, sel; };
__device__ __forceinline__ PixTile pix_tile(const PpConvArgs &a, int pt) {
    int sel = 0;
    for (int q = 1; q < a.nseg; ++q) if (pt >= a.seg[q].tile_begin) sel = q;
    const int lt = pt - a.seg[sel].tile_begin;
    const int nb = lt / a.seg[sel].h_blocks;
    return {nb * a.seg[sel].bn, (lt - nb * a.seg[sel].h_blocks) * a.seg[sel].bh, a.seg[sel].w0, sel};
}

template <int BN>
__global__ void __launch_bounds__(kPpThreads, 1)
conv_fprop_pp_kernel(const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmX0,
                     const __grid_constant__ CUtensorMap tmX1, const __grid_constant__ CUtensorMap tmX2,
                     const __grid_constant__ CUtensorMap tmX3, const __grid_constant__ CUtensorMap tmY0,
                     const __grid_constant__ CUtensorMap tmY1, const __grid_constant__ CUtensorMap tmY2,
                     const __grid_constant__ CUtensorMap tmY3, const __grid_constant__ PpConvArgs a) {
    using L = PpSmem<BN>;
    constexpr int STAGES = L::STAGES;
    extern __shared__ unsigned char smem_raw[];
    unsigned char *smem = (unsigned char *)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint64_t *full = (uint64_t *)(smem + L::BAR_OFF);
    uint64_t *empty = full + STAGES;
    const int wg = threadIdx.x >> 7;
    const int cchunks = a.C / BK;
    const int nkb = a.kh * a.kw * cchunks;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmB);
        tma_prefetch_desc(&tmX0);
        tma_prefetch_desc(&tmY0);
        for (int s = 0; s < STAGES; ++s) { mbar_init(full + s, 1); mbar_init(empty + s, 1); }
        fence_barrier_init();
    }
    __syncthreads();

    if (wg == 0) {
        // ------------------------------------------------------------ producer
        reg_dec<kPpProducerRegs>();
        if (threadIdx.x < 32 && elect_one()) {
            uint32_t it = 0;                                   // K blocks issued so far = ring position
            for (int t = blockIdx.x; t < a.tiles; t += gridDim.x) {
                const int pt = t / a.cout_tiles;
                const int n0 = (t - pt * a.cout_tiles) * BN;
                const PixTile p = pix_tile(a, pt);
                const CUtensorMap *tmX = p.sel == 0 ? &tmX0 : (p.sel == 1 ? &tmX1 : (p.sel == 2 ? &tmX2 : &tmX3));
                int cc = 0, ti = 0, tj = 0;
                for (int i = 0; i < nkb; ++i, ++it) {
                    const int s = it % STAGES;
                    mbar_wait(empty + s, ((it / STAGES) & 1) ^ 1);
                    unsigned char *dst = smem + s * L::STAGE_BYTES;
                    mbar_expect_tx(full + s, L::STAGE_BYTES);
                    tma_load_4d(tmX, full + s, dst, cc * BK, p.w0 + tj - a.pw, p.h0 + ti - a.ph, p.n);
                    tma_load_2d(&tmB, full + s, dst + L::A_BYTES, i * BK, n0);
                    if (++cc == cchunks) { cc = 0; if (++tj == a.kw) { tj = 0; ++ti; } }
                }
            }
        }
        return;
    }

    // ---------------------------------------------------------------- consumers
    reg_inc<kPpConsumerRegs>();
    const int c = wg - 1;                                      // consumer 0 takes the CTA's even tiles, 1 the odd ones
    const int mt = threadIdx.x & 127;
    const int w = mt >> 5, l = mt & 31;
    const int ntiles = (a.tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;   // >= 1: grid <= tiles
    const int turns0 = (ntiles + 1) >> 1;                      // consumer 0's tiles; consumer 1 has turns0 or turns0 - 1
    const int mine = (ntiles - c + 1) >> 1;
    unsigned char *out = smem + L::OUT_OFF + c * L::OUT_BYTES;
    const uint32_t out_addr = smem_u32(out);
    for (int j = 0; j < mine; ++j) {
        const int k = 2 * j + c;                               // the CTA's k-th tile
        // Order barrier: consumer 0's main loop of turn j follows consumer 1's of turn j - 1, and consumer 1's of turn j
        // follows consumer 0's of turn j.  Every sync has exactly one matching arrive.
        if (c == 0) { if (j > 0) named_bar_sync<256>(kBarTurn0); }
        else named_bar_sync<256>(kBarTurn1);
        const uint32_t it0 = (uint32_t)k * nkb;                // ring position of the tile's first K block
        AccTile<BN> acc;
        for (int i = 0; i < nkb; ++i) {
            const uint32_t it = it0 + i;
            const int s = it % STAGES;
            mbar_wait(full + s, (it / STAGES) & 1);
            wgmma_fence();
            const uint32_t a_addr = smem_u32(smem + s * L::STAGE_BYTES);
            const uint32_t b_addr = a_addr + L::A_BYTES;
#pragma unroll
            for (int kk = 0; kk < BK / WGMMA_K; ++kk)
                acc.template mma<0, 0>(desc_kmajor(a_addr, kk), desc_kmajor(a_addr, kk, 1), desc_kmajor(b_addr, kk),
                                       (i | kk) != 0);
            wgmma_commit();
            wgmma_wait<1>();                                   // block i - 1 has retired: hand its stage back
            if (i > 0 && mt == 0) mbar_arrive(empty + (it - 1) % STAGES);
        }
        if (c == 0) named_bar_arrive<256>(kBarTurn1);
        else if (j + 1 < turns0) named_bar_arrive<256>(kBarTurn0);
        wgmma_wait<0>();
        if (mt == 0) mbar_arrive(empty + (it0 + nkb - 1) % STAGES);

        // ------------------------------------------------------------ epilogue: fragments -> bf16 tile -> TMA store
        const int t = (int)blockIdx.x + k * (int)gridDim.x;
        const int pt = t / a.cout_tiles;
        const int n0 = (t - pt * a.cout_tiles) * BN;
        if (mt == 0) bulk_wait_group_read<0>();                // the previous tile's stores have read the staging tile
        named_bar_sync<128>(kBarEpi0 + c);
        // slice q = columns 64q..64q+63: row r at r * 128 B, 16-byte chunk j at (j ^ (r & 7)) (the 128-byte swizzle of the
        // store box).  Fragment d[half][4j + 2h + e] is row half * 64 + 16 w + l / 4 + 8 h, column 8 j + 2 (l % 4) + e, so
        // the 8x8 block (j, h) is one stmatrix operand; lanes 8i..8i+7 address block (j + i / 2, h = i % 2).
        const int sub = l >> 3, rr = l & 7;
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            const int row = half * 64 + 16 * w + 8 * (sub & 1) + rr;
#pragma unroll
            for (int j = 0; j < BN / 8; j += 2) {
                const int q = j >> 3, chunk = (j & 7) + (sub >> 1);
                const uint32_t addr = out_addr + q * L::SLICE_BYTES + row * 128 + ((chunk ^ (row & 7)) << 4);
                uint32_t r[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    __nv_bfloat162 h2 = __floats2bfloat162_rn(acc.d[half][4 * j + 2 * e], acc.d[half][4 * j + 2 * e + 1]);
                    r[e] = *reinterpret_cast<uint32_t *>(&h2);
                }
                stmatrix_x4(addr, r[0], r[1], r[2], r[3]);
            }
        }
        fence_proxy_async();                                   // generic-proxy smem writes -> visible to the TMA store
        named_bar_sync<128>(kBarEpi0 + c);
        if (mt == 0) {
            const PixTile p = pix_tile(a, pt);
            const CUtensorMap *tmY = p.sel == 0 ? &tmY0 : (p.sel == 1 ? &tmY1 : (p.sel == 2 ? &tmY2 : &tmY3));
#pragma unroll
            for (int q = 0; q < BN / 64; ++q)
                if (n0 + 64 * q < a.Cout) tma_store_4d(tmY, out + q * L::SLICE_BYTES, n0 + 64 * q, p.w0, p.h0, p.n);
            bulk_commit_group();
        }
    }
    if (c == 1 && mine < turns0) named_bar_sync<256>(kBarTurn1);   // consumer 0's last arrive
    if (mt == 0) bulk_wait_group<0>();                         // the staging tile must outlive the last store's reads
}

// =====================================================================================================
// Persistent implicit-GEMM weight gradient:  dW[co, tap*C + c] += sum_p dz[p, co] * x[pixel(p) shifted by tap, c]
//
// CTA tile 128 (Cout) x 256 (kh*kw*C columns): both consumer warpgroups read the same dz (A) stage and each owns one
// 128-column half of the x (B) operand, so a stage of dz is loaded once per 256 columns.  Both operands come MN-major by
// 4-D TMA exactly as in conv_wgrad_tcgen05_kernel (K block = RB output pixels of one row; tap shift = signed coordinate
// offset, padding = TMA zero fill).  The work is split stream-K: the iterations of the whole problem, ordered as (split,
// tile, K block of the split), are cut into gridDim.x equal contiguous ranges, one per CTA, so every SM gets the same number
// of K blocks whatever the tile count.  With splits ~ gridDim.x / tiles the CTAs that run side by side work on the same
// split, i.e. on the same rows of dz and x, which are then read from HBM once and hit in L2 by the other tiles.  A CTA accumulates each tile's part of its range in registers and adds it into dW (pre-zeroed by the caller)
// straight from the fragments with red.global.add.v4.f32.
// =====================================================================================================
struct PpWgradArgs {
    int C, Cout, K, kw, ph, pw, Ho, wboxes;
    int kb_total, n_tiles, tiles;     // K blocks per tile; 256-column tiles per 128-row block; all tiles
    int kb_split;                     // K blocks per split
    int total, per;                   // splits x tiles x kb_split iterations, per CTA
};

// The part of [g, g_end) that lies in one (split, tile): K blocks [kb_lo, kb_hi) of `tile` (empty past the last K block of
// a short last split) and the `len` iterations it spans.
struct WgradSeg { int tile, kb_lo, kb_hi, len; };
__device__ __forceinline__ WgradSeg wgrad_seg(const PpWgradArgs &a, int g, int g_end) {
    const int u = g / a.kb_split, kk = g - u * a.kb_split;
    const int sp = u / a.tiles;
    const int len = min(a.kb_split - kk, g_end - g);
    const int lo = sp * a.kb_split + kk;
    return {u - sp * a.tiles, min(lo, a.kb_total), min(lo + len, a.kb_total), len};
}

template <int RB> struct PpWgradSmem {
    static constexpr int STAGES = RB == 64 ? 4 : 3;
    static constexpr int ATOM = RB * 128;                  // one 64-wide MN atom: RB K rows of 128 B
    static constexpr int A_BYTES = 2 * ATOM;               // 128 output channels
    static constexpr int B_BYTES = 4 * ATOM;               // 256 columns
    static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
    static constexpr int BAR_OFF = STAGES * STAGE_BYTES;
    static constexpr int TOTAL = BAR_OFF + 2 * STAGES * 8 + 1024;
    static_assert(TOTAL <= 232448, "227 KB of opt-in shared memory");
};

__device__ __forceinline__ void red_add_v4(float *p, float a, float b, float c, float d) {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

template <int RB>
__global__ void __launch_bounds__(kPpThreads, 1)
conv_wgrad_pp_kernel(const __grid_constant__ CUtensorMap tmDz, const __grid_constant__ CUtensorMap tmX,
                     float *__restrict__ dW, const __grid_constant__ PpWgradArgs a) {
    using L = PpWgradSmem<RB>;
    constexpr int STAGES = L::STAGES;
    extern __shared__ unsigned char smem_raw[];
    unsigned char *smem = (unsigned char *)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint64_t *full = (uint64_t *)(smem + L::BAR_OFF);
    uint64_t *empty = full + STAGES;
    const int wg = threadIdx.x >> 7;
    const int g_begin = (int)blockIdx.x * a.per;
    const int g_end = min(a.total, g_begin + a.per);

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmDz);
        tma_prefetch_desc(&tmX);
        for (int s = 0; s < STAGES; ++s) { mbar_init(full + s, 1); mbar_init(empty + s, 2); }   // empty: both consumers
        fence_barrier_init();
    }
    __syncthreads();

    if (wg == 0) {
        // ------------------------------------------------------------ producer
        reg_dec<kPpProducerRegs>();
        if (threadIdx.x < 32 && elect_one()) {
            uint32_t it = 0;
            for (int g = g_begin; g < g_end;) {
                const WgradSeg sg = wgrad_seg(a, g, g_end);
                g += sg.len;
                const int tile = sg.tile, kb_lo = sg.kb_lo, kb_hi = sg.kb_hi;
                const int mt = tile / a.n_tiles;
                const int m0 = mt * BM, n0 = (tile - mt * a.n_tiles) * 256;
                int at_i[4], at_j[4], at_c[4];                 // the 4 column atoms of this tile: (tap, channel offset)
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const int col = n0 + 64 * q;
                    const int tap = col / a.C;
                    at_c[q] = col - tap * a.C;
                    at_i[q] = tap / a.kw;
                    at_j[q] = tap - at_i[q] * a.kw;
                }
                for (int kb = kb_lo; kb < kb_hi; ++kb, ++it) {
                    const int s = it % STAGES;
                    mbar_wait(empty + s, ((it / STAGES) & 1) ^ 1);
                    int r = kb;
                    const int wb = r % a.wboxes; r /= a.wboxes;
                    const int ho = r % a.Ho;
                    const int n = r / a.Ho;
                    unsigned char *a_dst = smem + s * L::STAGE_BYTES;
                    unsigned char *b_dst = a_dst + L::A_BYTES;
                    mbar_expect_tx(full + s, L::STAGE_BYTES);
                    tma_load_4d(&tmDz, full + s, a_dst, m0, wb * RB, ho, n);
                    tma_load_4d(&tmDz, full + s, a_dst + L::ATOM, m0 + 64, wb * RB, ho, n);
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        if (n0 + 64 * q < a.K)
                            tma_load_4d(&tmX, full + s, b_dst + q * L::ATOM, at_c[q], wb * RB + at_j[q] - a.pw,
                                        ho + at_i[q] - a.ph, n);
                        else   // column atom beyond kh*kw*C: keep the transaction count with an all-out-of-bounds box
                            tma_load_4d(&tmX, full + s, b_dst + q * L::ATOM, 0, -RB - 8, 0, n);
                    }
                }
            }
        }
        return;
    }

    // ---------------------------------------------------------------- consumers: column half c of every tile
    reg_inc<kPpConsumerRegs>();
    const int c = wg - 1;
    const int mt_ = threadIdx.x & 127;
    const int w = mt_ >> 5, l = mt_ & 31;
    const bool odd = l & 1;
    uint32_t it = 0;
    for (int g = g_begin; g < g_end;) {
        const WgradSeg sg = wgrad_seg(a, g, g_end);
        g += sg.len;
        const int tile = sg.tile, nkb = sg.kb_hi - sg.kb_lo;
        if (nkb == 0) continue;
        const int mt = tile / a.n_tiles;
        const int m0 = mt * BM, n0 = (tile - mt * a.n_tiles) * 256 + c * 128;
        AccTile<128> acc;
        for (int i = 0; i < nkb; ++i, ++it) {
            const int s = it % STAGES;
            mbar_wait(full + s, (it / STAGES) & 1);
            wgmma_fence();
            const uint32_t a_addr = smem_u32(smem + s * L::STAGE_BYTES);
            const uint32_t b_addr = a_addr + L::A_BYTES + c * 2 * L::ATOM;
#pragma unroll
            for (int k = 0; k < RB / WGMMA_K; ++k)
                acc.template mma<1, 1>(desc_mnmajor(a_addr, k, L::ATOM), desc_mnmajor(a_addr, k, L::ATOM, 1),
                                       desc_mnmajor(b_addr, k, L::ATOM), (i | k) != 0);
            wgmma_commit();
            wgmma_wait<1>();
            if (i > 0 && mt_ == 0) mbar_arrive(empty + (it - 1) % STAGES);
        }
        wgmma_wait<0>();
        if (mt_ == 0) mbar_arrive(empty + (it - 1) % STAGES);
        // Fragment d[half][4j + 2h + e] is row half * 64 + 16 w + l / 4 + 8 h, column 8 j + 2 (l % 4) + e.  Lanes l and
        // l ^ 1 swap a pair so that the even lane holds 4 consecutive columns of row h = 0 and the odd lane of row h = 1.
        const int col0 = n0 + 2 * (l & 3) - (odd ? 2 : 0);
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            const int row = m0 + half * 64 + 16 * w + (l >> 2) + (odd ? 8 : 0);
            float *dst = dW + (int64_t)row * a.K + col0;
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const float *d = &acc.d[half][4 * j];
                const float r0 = __shfl_xor_sync(0xffffffffu, odd ? d[0] : d[2], 1);
                const float r1 = __shfl_xor_sync(0xffffffffu, odd ? d[1] : d[3], 1);
                if (row < a.Cout && col0 + 8 * j < a.K) {
                    if (odd) red_add_v4(dst + 8 * j, r0, r1, d[2], d[3]);
                    else red_add_v4(dst + 8 * j, d[0], d[1], r0, r1);
                }
            }
        }
    }
}

template <int BN>
int launch_pp(const CUtensorMap &tb, const CUtensorMap *tx, const CUtensorMap *ty, const PpConvArgs &a, int grid,
              cudaStream_t st) {
    auto kern = conv_fprop_pp_kernel<BN>;
    { int rc = ensure_dyn_smem((const void *)kern, PpSmem<BN>::TOTAL, "conv_fprop_pp smem attr"); if (rc) return rc; }
    kern<<<grid, kPpThreads, PpSmem<BN>::TOTAL, st>>>(tb, tx[0], tx[1], tx[2], tx[3], ty[0], ty[1], ty[2], ty[3], a);
    return check_launch("conv_fprop_pp_kernel");
}

template <int RB>
int launch_wgrad_pp(const CUtensorMap &tdz, const CUtensorMap &tx, float *dW, const PpWgradArgs &a, int grid,
                    cudaStream_t st) {
    auto kern = conv_wgrad_pp_kernel<RB>;
    { int rc = ensure_dyn_smem((const void *)kern, PpWgradSmem<RB>::TOTAL, "conv_wgrad_pp smem attr"); if (rc) return rc; }
    kern<<<grid, kPpThreads, PpWgradSmem<RB>::TOTAL, st>>>(tdz, tx, dW, a);
    return check_launch("conv_wgrad_pp_kernel");
}

}  // namespace

extern "C" {

/* Persistent ping-pong implicit-GEMM stride-1 convolution on NHWC bf16: y[N*Ho*Wo, Cout] bf16 = conv(x[N,H,W,C],
 * Wm[Cout, kh*kw*C]); no bias, no activation.  With flipped/transposed weights and padding (k-1-p) it is the input
 * gradient.  Bit-identical to mr_conv_fprop_tcgen05 with a bf16 output.  MR_ERR_UNSUPPORTED unless C % 64 == 0,
 * Cout % 8 == 0, the pointers are 16-byte aligned and the output tiles with at most four TMA box segments. */
int mr_conv_fprop_pp(const void *x, const void *Wm, void *y, int N, int H, int W, int C, int Cout, int kh, int kw, int ph,
                     int pw, void *stream) {
    if (N < 0 || H <= 0 || W <= 0 || C <= 0 || Cout <= 0 || kh <= 0 || kw <= 0 || ph < 0 || pw < 0) return MR_ERR_BAD_SHAPE;
    const int Ho = H + 2 * ph - kh + 1, Wo = W + 2 * pw - kw + 1;
    if (Ho <= 0 || Wo <= 0) return MR_ERR_BAD_SHAPE;
    if (N == 0) return MR_OK;
    if (!x || !Wm || !y) return MR_ERR_NULL_POINTER;
    if (C % 64 || Cout % 8 || ((uintptr_t)x % 16) || ((uintptr_t)Wm % 16) || ((uintptr_t)y % 16)) return MR_ERR_UNSUPPORTED;
    if ((int64_t)N * Ho * Wo > (1LL << 31) - 256) return MR_ERR_UNSUPPORTED;
    PpConvArgs a;
    a.C = C; a.Cout = Cout; a.kh = kh; a.kw = kw; a.ph = ph; a.pw = pw;
    CUtensorMap tx[kMaxConvSegs], ty[kMaxConvSegs];
    int pixel_tiles = 0;
    int rc = plan_conv_segments(x, N, H, W, C, Ho, Wo, 1, 1, a.seg, tx, &a.nseg, &pixel_tiles);
    if (rc) return rc;
    if (a.nseg == 0) return MR_ERR_UNSUPPORTED;
    for (int q = 0; q < a.nseg; ++q) {
        rc = make_map_nhwc(&ty[q], y, Cout, Wo, Ho, N, a.seg[q].bw, a.seg[q].bh, a.seg[q].bn);
        if (rc) return rc;
    }
    for (int q = a.nseg; q < kMaxConvSegs; ++q) { tx[q] = tx[0]; ty[q] = ty[0]; }
    const int BN = Cout > 64 ? 128 : 64;
    const int64_t K = (int64_t)kh * kw * C;
    CUtensorMap tb;
    rc = make_map(&tb, Wm, K, Cout, K, BK, BN);
    if (rc) return rc;
    a.cout_tiles = (int)ceil_div(Cout, BN);
    const int64_t tiles = (int64_t)pixel_tiles * a.cout_tiles;
    if (tiles > (1LL << 31) - 1) return MR_ERR_UNSUPPORTED;
    a.tiles = (int)tiles;
    const int sms = sm_count();
    if (sms <= 0) { set_cuda_error(cudaErrorUnknown, "multiprocessor count"); return MR_ERR_CUDA; }
    const int grid = (int)(tiles < sms ? tiles : sms);
    cudaStream_t st = (cudaStream_t)stream;
    return BN == 128 ? launch_pp<128>(tb, tx, ty, a, grid, st) : launch_pp<64>(tb, tx, ty, a, grid, st);
}

/* Persistent implicit-GEMM weight gradient, stride 1: dWm[Cout, kh*kw*C] fp32 (ACCUMULATED atomically: zero it first) from
 * dz[N,Ho,Wo,Cout] and x[N,H,W,C] (NHWC bf16).  The tiles' K blocks are split evenly over `ctas` CTAs (clamped to
 * [1, min(SM count, K blocks)]).  MR_ERR_UNSUPPORTED unless C % 64 == 0, Cout % 8 == 0 and 16-byte aligned operands. */
int mr_conv_wgrad_pp(const void *dz, const void *x, float *dWm, int N, int H, int W, int C, int Cout, int kh, int kw, int ph,
                     int pw, int ctas, void *stream) {
    if (N < 0 || H <= 0 || W <= 0 || C <= 0 || Cout <= 0 || kh <= 0 || kw <= 0 || ph < 0 || pw < 0) return MR_ERR_BAD_SHAPE;
    const int Ho = H + 2 * ph - kh + 1, Wo = W + 2 * pw - kw + 1;
    if (Ho <= 0 || Wo <= 0) return MR_ERR_BAD_SHAPE;
    if (N == 0) return MR_OK;
    if (!dz || !x || !dWm) return MR_ERR_NULL_POINTER;
    if (C % 64 || Cout % 8 || ((uintptr_t)x % 16) || ((uintptr_t)dz % 16) || ((uintptr_t)dWm % 16)) return MR_ERR_UNSUPPORTED;
    const bool rb80 = Wo > 64 && Wo <= 80;
    const int RB = rb80 ? 80 : 64;
    PpWgradArgs a;
    a.C = C; a.Cout = Cout; a.K = kh * kw * C; a.kw = kw; a.ph = ph; a.pw = pw; a.Ho = Ho;
    a.wboxes = (int)ceil_div(Wo, RB);
    a.n_tiles = (int)ceil_div(a.K, 256);
    const int64_t kb_total = (int64_t)N * Ho * a.wboxes;
    const int64_t tiles = ceil_div(Cout, BM) * a.n_tiles;
    if (kb_total * tiles > (1LL << 31) / 2) return MR_ERR_UNSUPPORTED;
    a.kb_total = (int)kb_total;
    a.tiles = (int)tiles;
    const int sms = sm_count();
    if (ctas <= 0 || ctas > sms) ctas = sms;
    if (ctas > kb_total * tiles) ctas = (int)(kb_total * tiles);
    const int splits = (int)std::min<int64_t>(kb_total, std::max<int64_t>(1, ctas / tiles));
    /* When splits x tiles CTAs still fill 90 % of the requested ones, give each CTA exactly one (split, tile): the CTAs
     * then all sit at the same K offset of their split and read the same dz / x rows at the same time. */
    if (splits > 1 && (int64_t)splits * tiles * 10 >= (int64_t)ctas * 9) ctas = splits * (int)tiles;
    a.kb_split = (int)ceil_div(kb_total, splits);
    a.total = splits * a.tiles * a.kb_split;
    a.per = (int)ceil_div(a.total, ctas);
    const int grid = (int)ceil_div(a.total, a.per);
    CUtensorMap tdz, tx;
    int rc = make_map_nhwc(&tdz, dz, Cout, Wo, Ho, N, RB);
    if (rc) return rc;
    rc = make_map_nhwc(&tx, x, C, W, H, N, RB);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    return rb80 ? launch_wgrad_pp<80>(tdz, tx, dWm, a, grid, st) : launch_wgrad_pp<64>(tdz, tx, dWm, a, grid, st);
}

}  // extern "C"
