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
#include <numeric>

namespace {

constexpr int kPpThreads = 384;
constexpr int kPpProducerRegs = 40;
constexpr int kPpConsumerRegs = 232;       // 128 * 40 + 256 * 232 <= 65536
static_assert(128 * kPpProducerRegs + 256 * kPpConsumerRegs <= 65536, "register file");

// Named barriers (0 is __syncthreads): the consumers' turn barriers, and one per consumer for its epilogue.
constexpr int kBarTurn0 = 1, kBarTurn1 = 2, kBarEpi0 = 3;

// K blocks (64 deep) from which mr_conv_fprop_pp picks conv_fprop_m256_kernel over conv_fprop_pp_kernel.  On an H100 SXM
// the 256-pixel tiles were faster at 36 K blocks (L3 forward, L2 input gradient at batch 512) and 2 % slower at 32 (L6
// forward), where the ping-pong kernel's overlap of one consumer's epilogue with the other's main loop matters more.
constexpr int kM256MinKb = 36;

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
    int pix_tiles, cout_tiles, tiles; // tiles = 128-pixel tiles (pairs of them for conv_fprop_m256_kernel) x cout_tiles
    int halo;                         // conv_fprop_pp_kernel: halo mode (PpHaloSmem), tmX0 is the halo map
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

// One consumer's 128 x BN fp32 accumulator -> its bf16 staging tile (BN/64 slices of 128 rows x 128 B, the TMA store boxes):
// row r at r * 128 B, 16-byte chunk j at (j ^ (r & 7)) (the 128-byte swizzle of the store box).  Fragment d[half][4j + 2h
// + e] is row half * 64 + 16 w + l / 4 + 8 h, column 8 j + 2 (l % 4) + e, so the 8x8 block (j, h) is one stmatrix operand;
// lanes 8i..8i+7 address block (j + i / 2, h = i % 2).
template <int BN>
__device__ __forceinline__ void pp_stage_tile(const AccTile<BN> &acc, uint32_t out_addr, int w, int l) {
    constexpr int SLICE_BYTES = BM * 64 * 2;
    const int sub = l >> 3, rr = l & 7;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
        const int row = half * 64 + 16 * w + 8 * (sub & 1) + rr;
#pragma unroll
        for (int j = 0; j < BN / 8; j += 2) {
            const int q = j >> 3, chunk = (j & 7) + (sub >> 1);
            const uint32_t addr = out_addr + q * SLICE_BYTES + row * 128 + ((chunk ^ (row & 7)) << 4);
            uint32_t r[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                __nv_bfloat162 h2 = __floats2bfloat162_rn(acc.d[half][4 * j + 2 * e], acc.d[half][4 * j + 2 * e + 1]);
                r[e] = *reinterpret_cast<uint32_t *>(&h2);
            }
            stmatrix_x4(addr, r[0], r[1], r[2], r[3]);
        }
    }
}

// Halo mode of conv_fprop_pp_kernel, for calls whose every pixel tile is one whole 128-pixel output row (bw = 128,
// bh = bn = 1: L1's forward and input gradient at W = 128): the kw taps of a tap row then read the same 128 + kw - 1
// input pixels, one 128-byte smem row further per tap.  The producer loads that halo once per (tap row, channel block),
// with the first tap's weight block and on its full barrier, into one of SLOTS halo slots; the consumer takes K block
// (i, j, cb) from halo slot (i, cb) with the A descriptor j rows into it and releases the slot after its last tap.  K
// order (tap-major, 64-channel blocks inner) and the instruction sequence are those of the normal mode, so the output is
// the same bits, with a third of the activation bytes from L2 at kw = 3.  SLOTS >= C / 64, or the first tap of a row would
// wait for a slot its own row holds.
constexpr int kHaloSlots = 4, kHaloMaxKw = 8;
template <int BN> struct PpHaloSmem {
    static constexpr int SLOT_BYTES = 17 * 1024;          // >= (128 + kHaloMaxKw - 1) * 128, 1024-byte aligned slots
    static constexpr int STAGES = BN == 128 ? 5 : 8;
    static constexpr int B_BYTES = BN * BK * 2;
    static constexpr int W_OFF = kHaloSlots * SLOT_BYTES;
    static constexpr int OUT_BYTES = PpSmem<BN>::OUT_BYTES;
    static constexpr int OUT_OFF = W_OFF + STAGES * B_BYTES;
    static constexpr int BAR_OFF = OUT_OFF + 2 * OUT_BYTES;
    static constexpr int TOTAL = BAR_OFF + (2 * STAGES + kHaloSlots) * 8 + 1024;
    static_assert((128 + kHaloMaxKw - 1) * 128 <= SLOT_BYTES && OUT_OFF % 1024 == 0, "halo layout");
    static_assert(TOTAL <= 232448, "227 KB of opt-in shared memory");
};

template <int BN>
__device__ __forceinline__ void pp_halo(const CUtensorMap &tmB, const CUtensorMap &tmH, const CUtensorMap &tmY0,
                                        const CUtensorMap &tmY1, const CUtensorMap &tmY2, const CUtensorMap &tmY3,
                                        const PpConvArgs &a) {
    using L = PpHaloSmem<BN>;
    constexpr int STAGES = L::STAGES, SLOTS = kHaloSlots;
    extern __shared__ unsigned char smem_raw[];
    unsigned char *smem = (unsigned char *)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint64_t *full = (uint64_t *)(smem + L::BAR_OFF);
    uint64_t *empty = full + STAGES;
    uint64_t *hempty = empty + STAGES;
    const int wg = threadIdx.x >> 7;
    const int cchunks = a.C / BK;
    const int nkb = a.kh * a.kw * cchunks;
    const int hrow = a.kh * cchunks;                           // halos per tile

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmB);
        tma_prefetch_desc(&tmH);
        tma_prefetch_desc(&tmY0);
        for (int s = 0; s < STAGES; ++s) { mbar_init(full + s, 1); mbar_init(empty + s, 1); }
        for (int s = 0; s < SLOTS; ++s) mbar_init(hempty + s, 1);
        fence_barrier_init();
    }
    __syncthreads();

    if (wg == 0) {
        // ------------------------------------------------------------ producer
        reg_dec<kPpProducerRegs>();
        if (threadIdx.x < 32 && elect_one()) {
            const uint32_t halo_bytes = (128 + a.kw - 1) * 128;
            uint32_t it = 0, hs = 0;                           // K blocks and halos issued so far
            for (int t = blockIdx.x; t < a.tiles; t += gridDim.x) {
                const int pt = t / a.cout_tiles;
                const int n0 = (t - pt * a.cout_tiles) * BN;
                const PixTile p = pix_tile(a, pt);
                int cc = 0, ti = 0, tj = 0;
                for (int i = 0; i < nkb; ++i, ++it) {
                    const int s = it % STAGES;
                    mbar_wait(empty + s, ((it / STAGES) & 1) ^ 1);
                    if (tj == 0) {
                        const int h = hs % SLOTS;
                        mbar_wait(hempty + h, ((hs / SLOTS) & 1) ^ 1);
                        mbar_expect_tx(full + s, L::B_BYTES + halo_bytes);
                        tma_load_4d(&tmH, full + s, smem + h * L::SLOT_BYTES, cc * BK, p.w0 - a.pw, p.h0 + ti - a.ph, p.n);
                        ++hs;
                    } else {
                        mbar_expect_tx(full + s, L::B_BYTES);
                    }
                    tma_load_2d(&tmB, full + s, smem + L::W_OFF + s * L::B_BYTES, i * BK, n0);
                    if (++cc == cchunks) { cc = 0; if (++tj == a.kw) { tj = 0; ++ti; } }
                }
            }
        }
        return;
    }

    // ---------------------------------------------------------------- consumers: as conv_fprop_pp_kernel's
    reg_inc<kPpConsumerRegs>();
    const int c = wg - 1;
    const int mt = threadIdx.x & 127;
    const int w = mt >> 5, l = mt & 31;
    const int ntiles = (a.tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
    const int turns0 = (ntiles + 1) >> 1;
    const int mine = (ntiles - c + 1) >> 1;
    unsigned char *out = smem + L::OUT_OFF + c * L::OUT_BYTES;
    const uint32_t out_addr = smem_u32(out);
    const uint32_t halo_addr = smem_u32(smem);
    const uint32_t w_addr = smem_u32(smem + L::W_OFF);
    for (int j = 0; j < mine; ++j) {
        const int k = 2 * j + c;
        if (c == 0) { if (j > 0) named_bar_sync<256>(kBarTurn0); }
        else named_bar_sync<256>(kBarTurn1);
        const uint32_t it0 = (uint32_t)k * nkb;
        const uint32_t hs0 = (uint32_t)k * hrow;               // the tile's first halo
        AccTile<BN> acc;
        int cc = 0, ti = 0, tj = 0;
        int prev_slot = 0;                                     // block i - 1's halo slot, released after its last tap
        bool prev_last = false;
        for (int i = 0; i < nkb; ++i) {
            const uint32_t it = it0 + i;
            const int s = it % STAGES;
            const int h = (hs0 + ti * cchunks + cc) % SLOTS;
            mbar_wait(full + s, (it / STAGES) & 1);
            wgmma_fence();
            const uint32_t a_addr = halo_addr + h * L::SLOT_BYTES + tj * 128;
            const uint32_t b_addr = w_addr + s * L::B_BYTES;
            // The descriptor starts tj 128-byte rows into the 1024-byte aligned slot with matrix base offset 0: wgmma
            // applies the 128-byte swizzle to the absolute shared address, as the TMA did when it wrote the halo (a base
            // offset of (a_addr >> 7) & 7 shifts the pattern a second time and gives wrong sums).
#pragma unroll
            for (int kk = 0; kk < BK / WGMMA_K; ++kk)
                acc.template mma<0, 0>(desc_kmajor(a_addr, kk), desc_kmajor(a_addr, kk, 1), desc_kmajor(b_addr, kk),
                                       (i | kk) != 0);
            wgmma_commit();
            wgmma_wait<1>();
            if (i > 0 && mt == 0) {
                mbar_arrive(empty + (it - 1) % STAGES);
                if (prev_last) mbar_arrive(hempty + prev_slot);
            }
            prev_slot = h;
            prev_last = tj == a.kw - 1;
            if (++cc == cchunks) { cc = 0; if (++tj == a.kw) { tj = 0; ++ti; } }
        }
        if (c == 0) named_bar_arrive<256>(kBarTurn1);
        else if (j + 1 < turns0) named_bar_arrive<256>(kBarTurn0);
        wgmma_wait<0>();
        if (mt == 0) { mbar_arrive(empty + (it0 + nkb - 1) % STAGES); mbar_arrive(hempty + prev_slot); }

        const int t = (int)blockIdx.x + k * (int)gridDim.x;
        const int pt = t / a.cout_tiles;
        const int n0 = (t - pt * a.cout_tiles) * BN;
        if (mt == 0) bulk_wait_group_read<0>();
        named_bar_sync<128>(kBarEpi0 + c);
        pp_stage_tile<BN>(acc, out_addr, w, l);
        fence_proxy_async();
        named_bar_sync<128>(kBarEpi0 + c);
        if (mt == 0) {
            const PixTile p = pix_tile(a, pt);
            const CUtensorMap *tmY = p.sel == 0 ? &tmY0 : (p.sel == 1 ? &tmY1 : (p.sel == 2 ? &tmY2 : &tmY3));
#pragma unroll
            for (int q = 0; q < BN / 64; ++q)
                if (n0 + 64 * q < a.Cout) tma_store_4d(tmY, out + q * BM * 128, n0 + 64 * q, p.w0, p.h0, p.n);
            bulk_commit_group();
        }
    }
    if (c == 1 && mine < turns0) named_bar_sync<256>(kBarTurn1);
    if (mt == 0) bulk_wait_group<0>();
}

template <int BN>
__global__ void __launch_bounds__(kPpThreads, 1)
conv_fprop_pp_kernel(const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmX0,
                     const __grid_constant__ CUtensorMap tmX1, const __grid_constant__ CUtensorMap tmX2,
                     const __grid_constant__ CUtensorMap tmX3, const __grid_constant__ CUtensorMap tmY0,
                     const __grid_constant__ CUtensorMap tmY1, const __grid_constant__ CUtensorMap tmY2,
                     const __grid_constant__ CUtensorMap tmY3, const __grid_constant__ PpConvArgs a) {
    if (a.halo) { pp_halo<BN>(tmB, tmX0, tmY0, tmY1, tmY2, tmY3, a); return; }
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
        pp_stage_tile<BN>(acc, out_addr, w, l);
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
// Large-K variant (kM256MinKb): a CTA tile is two consecutive 128-pixel tiles x one BN-wide Cout tile.  A stage holds both activation
// boxes (each from its own segment's tensor map) and ONE weight box, and consumer c multiplies activation box c by it, so
// the CTA loads 48 KB per 4.2 MFLOP instead of conv_fprop_pp_kernel's 32 KB per 2.1 MFLOP.  Each consumer's accumulator,
// K order, instruction sequence and epilogue are those of conv_fprop_pp_kernel<BN>: the output is the same bits.  Both
// consumers work on the same stage at once (its empty barrier takes two arrivals), so there is no turn order and no
// epilogue overlap inside the CTA; the producer keeps filling the ring while the consumers store.  An odd last pixel tile
// leaves consumer 1 without a tile: it stores nothing but still consumes every stage, whose second box the producer loads
// entirely out of bounds (zero fill) to keep the transaction count.
// =====================================================================================================
template <int BN> struct M256Smem {
    static constexpr int STAGES = 3;
    static constexpr int A_BYTES = BM * BK * 2;            // one 128-pixel activation box
    static constexpr int B_BYTES = BN * BK * 2;
    static constexpr int STAGE_BYTES = 2 * A_BYTES + B_BYTES;
    static constexpr int SLICE_BYTES = BM * 64 * 2;
    static constexpr int OUT_BYTES = (BN / 64) * SLICE_BYTES;
    static constexpr int OUT_OFF = STAGES * STAGE_BYTES;
    static constexpr int BAR_OFF = OUT_OFF + 2 * OUT_BYTES;
    static constexpr int TOTAL = BAR_OFF + 2 * STAGES * 8 + 1024;
    static_assert(TOTAL <= 232448, "227 KB of opt-in shared memory");
};

template <int BN>
__global__ void __launch_bounds__(kPpThreads, 1)
conv_fprop_m256_kernel(const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmX0,
                       const __grid_constant__ CUtensorMap tmX1, const __grid_constant__ CUtensorMap tmX2,
                       const __grid_constant__ CUtensorMap tmX3, const __grid_constant__ CUtensorMap tmY0,
                       const __grid_constant__ CUtensorMap tmY1, const __grid_constant__ CUtensorMap tmY2,
                       const __grid_constant__ CUtensorMap tmY3, const __grid_constant__ PpConvArgs a) {
    using L = M256Smem<BN>;
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
        for (int s = 0; s < STAGES; ++s) { mbar_init(full + s, 1); mbar_init(empty + s, 2); }   // empty: both consumers
        fence_barrier_init();
    }
    __syncthreads();

    if (wg == 0) {
        // ------------------------------------------------------------ producer
        reg_dec<kPpProducerRegs>();
        if (threadIdx.x < 32 && elect_one()) {
            uint32_t it = 0;
            for (int t = blockIdx.x; t < a.tiles; t += gridDim.x) {
                const int pair = t / a.cout_tiles;
                const int n0 = (t - pair * a.cout_tiles) * BN;
                const bool two = 2 * pair + 1 < a.pix_tiles;
                const PixTile p0 = pix_tile(a, 2 * pair);
                const PixTile p1 = two ? pix_tile(a, 2 * pair + 1) : p0;
                const CUtensorMap *tx0 = p0.sel == 0 ? &tmX0 : (p0.sel == 1 ? &tmX1 : (p0.sel == 2 ? &tmX2 : &tmX3));
                const CUtensorMap *tx1 = p1.sel == 0 ? &tmX0 : (p1.sel == 1 ? &tmX1 : (p1.sel == 2 ? &tmX2 : &tmX3));
                // no second tile: a box wholly left of the tensor (w + box width <= 0), all zero fill
                const int w1 = two ? p1.w0 - a.pw : -256;
                int cc = 0, ti = 0, tj = 0;
                for (int i = 0; i < nkb; ++i, ++it) {
                    const int s = it % STAGES;
                    mbar_wait(empty + s, ((it / STAGES) & 1) ^ 1);
                    unsigned char *dst = smem + s * L::STAGE_BYTES;
                    mbar_expect_tx(full + s, L::STAGE_BYTES);
                    tma_load_4d(tx0, full + s, dst, cc * BK, p0.w0 + tj - a.pw, p0.h0 + ti - a.ph, p0.n);
                    tma_load_4d(tx1, full + s, dst + L::A_BYTES, cc * BK, w1 + (two ? tj : 0), p1.h0 + ti - a.ph, p1.n);
                    tma_load_2d(&tmB, full + s, dst + 2 * L::A_BYTES, i * BK, n0);
                    if (++cc == cchunks) { cc = 0; if (++tj == a.kw) { tj = 0; ++ti; } }
                }
            }
        }
        return;
    }

    // ---------------------------------------------------------------- consumers: pixel tile c of every pair
    reg_inc<kPpConsumerRegs>();
    const int c = wg - 1;
    const int mt = threadIdx.x & 127;
    const int w = mt >> 5, l = mt & 31;
    unsigned char *out = smem + L::OUT_OFF + c * L::OUT_BYTES;
    const uint32_t out_addr = smem_u32(out);
    uint32_t it0 = 0;                                          // ring position of the tile's first K block
    for (int t = blockIdx.x; t < a.tiles; t += gridDim.x, it0 += nkb) {
        AccTile<BN> acc;
        for (int i = 0; i < nkb; ++i) {
            const uint32_t it = it0 + i;
            const int s = it % STAGES;
            mbar_wait(full + s, (it / STAGES) & 1);
            wgmma_fence();
            const uint32_t a_addr = smem_u32(smem + s * L::STAGE_BYTES + c * L::A_BYTES);
            const uint32_t b_addr = smem_u32(smem + s * L::STAGE_BYTES + 2 * L::A_BYTES);
#pragma unroll
            for (int kk = 0; kk < BK / WGMMA_K; ++kk)
                acc.template mma<0, 0>(desc_kmajor(a_addr, kk), desc_kmajor(a_addr, kk, 1), desc_kmajor(b_addr, kk),
                                       (i | kk) != 0);
            wgmma_commit();
            wgmma_wait<1>();                                   // block i - 1 has retired: hand its stage back
            if (i > 0 && mt == 0) mbar_arrive(empty + (it - 1) % STAGES);
        }
        wgmma_wait<0>();
        if (mt == 0) mbar_arrive(empty + (it0 + nkb - 1) % STAGES);

        // ------------------------------------------------------------ epilogue: as conv_fprop_pp_kernel's
        const int pair = t / a.cout_tiles;
        const int n0 = (t - pair * a.cout_tiles) * BN;
        const int pt = 2 * pair + c;
        if (pt >= a.pix_tiles) continue;                       // consumer 1 of an odd last pair
        if (mt == 0) bulk_wait_group_read<0>();                // the previous tile's stores have read the staging tile
        named_bar_sync<128>(kBarEpi0 + c);
        pp_stage_tile<BN>(acc, out_addr, w, l);
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
    if (mt == 0) bulk_wait_group<0>();                         // the staging tile must outlive the last store's reads
}

// =====================================================================================================
// Persistent implicit-GEMM weight gradient:  dW[co, tap*C + c] += sum_p dz[p, co] * x[pixel(p) shifted by tap, c]
//
// CTA tile 128 (Cout) x 256 (kh*kw*C columns): both consumer warpgroups read the same dz (A) stage and each owns one
// 128-column half of the x (B) operand, so a stage of dz is loaded once per 256 columns.  Both operands come MN-major by
// 4-D TMA (tap shift = signed coordinate offset, padding = TMA zero fill).  A K block is RB output pixels, the box
// bw columns x 1 row x bn images (bw * bn = RB) of one segment of the plan_wgrad_segments plan; dz and x are loaded with
// boxes of the same geometry, so row r of both operand tiles is the same output pixel and the order of the pixels does not
// matter.  The segments tile the output width exactly, so only a segment's last image block multiplies zero fill.  The K
// blocks are cut into `splits` equal splits; a unit is one (split, tile), and the units, numbered split-major, are handed
// out strided by gridDim.x.  The planner makes the unit count a whole multiple of the grid, so every CTA gets the same
// number of units, and the CTAs that run side by side work on one split or on adjacent ones, i.e. on the same images of dz
// and x, which are then read from HBM once and hit in L2 by the other tiles.  A CTA accumulates a unit in registers and
// adds it into dW (pre-zeroed by the caller) straight from the fragments with red.global.add.v4.f32.
// =====================================================================================================
// K-block segments of the weight gradient: columns [w0, w0 + w_blocks * bw) of the output, in boxes of bw x 1 x bn
// pixels; the segment's K blocks are numbered from kb_begin, box column fastest, then the output row, then the image block.
constexpr int kMaxWgradSegs = 5;
struct WgradSeg { int w0, bw, bn, w_blocks, kb_begin; };

struct PpWgradArgs {
    int C, Cout, K, kw, ph, pw, Ho;
    int nseg;
    WgradSeg seg[kMaxWgradSegs];
    int kb_total, n_tiles, tiles;     // K blocks per tile; column tiles per 128-row block; all tiles
    int kb_split;                     // K blocks per split (the last split may be shorter, or empty)
    int units;                        // splits x tiles
};
// One dz and one x tensor map per segment, with that segment's box.
struct WgradMaps { CUtensorMap dz[kMaxWgradSegs], x[kMaxWgradSegs]; };

// Output pixels per K block: 80 when 64 < Wo <= 80 (L4-L6 of the CRNN, Wo = 65 and 66), 64 otherwise.
__host__ __device__ constexpr int wgrad_rb(int Wo) { return Wo > 64 && Wo <= 80 ? 80 : 64; }

// The K-block segments of an [N, Ho, Wo] output.  RB = 80: the first floor(Wo / 16) * 16 columns in 16 x 1 x 5 boxes,
// then the rest in power-of-two widths bw = 8, 4, 2, 1, each in bw x 1 x (80 / bw) boxes (Wo = 65: 1,676 K blocks at
// L5 instead of the 2,048 of one 80-wide box per row, 99.3 % of them real pixels).  RB = 64: one segment of RB-wide row
// boxes.  -> the K-block total.
int64_t plan_wgrad_segments(int N, int Ho, int Wo, int RB, WgradSeg *seg, int *nseg) {
    int64_t kb = 0;
    *nseg = 0;
    auto add = [&](int w0, int bw, int w_blocks) {
        WgradSeg &s = seg[(*nseg)++];
        s.w0 = w0; s.bw = bw; s.bn = RB / bw; s.w_blocks = w_blocks; s.kb_begin = (int)kb;
        kb += (int64_t)w_blocks * Ho * ceil_div(N, s.bn);
    };
    if (RB == 80) {
        const int w16 = Wo / 16 * 16;
        add(0, 16, Wo / 16);
        for (int bw = 8, w0 = w16; bw >= 1; bw >>= 1)
            if ((Wo - w16) & bw) { add(w0, bw, 1); w0 += bw; }
    } else {
        add(0, RB, (int)ceil_div(Wo, RB));
    }
    return kb;
}

// Unit u = (split u / tiles, tile u % tiles): K blocks [kb_lo, kb_hi) of `tile`.
struct WgradUnit { int tile, kb_lo, kb_hi; };
__device__ __forceinline__ WgradUnit wgrad_unit(const PpWgradArgs &a, int u) {
    const int sp = u / a.tiles;
    const int lo = min(sp * a.kb_split, a.kb_total);
    return {u - sp * a.tiles, lo, min(lo + a.kb_split, a.kb_total)};
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

// The weight gradient's producer, run by one elected lane: every K block of every unit the CTA owns, as the two 64-row dz
// atoms of the 128-row tile and the NATOM 64-column x atoms of its NATOM * 64-column tile, through the ring of layout L
// (A: the dz atoms, then B: the x atoms, each L::ATOM bytes).
template <typename L, int NATOM>
__device__ __forceinline__ void wgrad_produce(const WgradMaps &tm, const PpWgradArgs &a, unsigned char *smem, uint64_t *full,
                                              uint64_t *empty) {
    constexpr int STAGES = L::STAGES;
    uint32_t it = 0;
    for (int u = blockIdx.x; u < a.units; u += gridDim.x) {
        const WgradUnit un = wgrad_unit(a, u);
        const int tile = un.tile, kb_lo = un.kb_lo, kb_hi = un.kb_hi;
        const int mt = tile / a.n_tiles;
        const int m0 = mt * BM, n0 = (tile - mt * a.n_tiles) * (64 * NATOM);
        int at_i[NATOM], at_j[NATOM], at_c[NATOM];     // the column atoms of this tile: (tap, channel offset)
#pragma unroll
        for (int q = 0; q < NATOM; ++q) {
            const int col = n0 + 64 * q;
            const int tap = col / a.C;
            at_c[q] = col - tap * a.C;
            at_i[q] = tap / a.kw;
            at_j[q] = tap - at_i[q] * a.kw;
        }
        if (kb_lo == kb_hi) continue;
        // The unit's first K block is decoded once; the loop then steps (column block, row, image block) and
        // the segment, so the segment's fields stay in registers off the path from a free stage to its loads.
        int sel = 0;
        for (int q = 1; q < a.nseg; ++q) if (kb_lo >= a.seg[q].kb_begin) sel = q;
        WgradSeg sg = a.seg[sel];
        int next = sel + 1 < a.nseg ? a.seg[sel + 1].kb_begin : a.kb_total;
        int r = kb_lo - sg.kb_begin;
        int wb = r % sg.w_blocks;
        r /= sg.w_blocks;
        int ho = r % a.Ho, n = r / a.Ho * sg.bn;
        const CUtensorMap *tdz = &tm.dz[sel], *tx = &tm.x[sel];
        for (int kb = kb_lo; kb < kb_hi; ++kb, ++it) {
            if (kb == next) {
                ++sel;
                sg = a.seg[sel];
                next = sel + 1 < a.nseg ? a.seg[sel + 1].kb_begin : a.kb_total;
                wb = 0; ho = 0; n = 0;
                tdz = &tm.dz[sel]; tx = &tm.x[sel];
            }
            const int s = it % STAGES;
            mbar_wait(empty + s, ((it / STAGES) & 1) ^ 1);
            const int w = sg.w0 + wb * sg.bw;
            unsigned char *a_dst = smem + s * L::STAGE_BYTES;
            unsigned char *b_dst = a_dst + L::A_BYTES;
            mbar_expect_tx(full + s, L::STAGE_BYTES);
            tma_load_4d(tdz, full + s, a_dst, m0, w, ho, n);
            tma_load_4d(tdz, full + s, a_dst + L::ATOM, m0 + 64, w, ho, n);
#pragma unroll
            for (int q = 0; q < NATOM; ++q) {
                if (n0 + 64 * q < a.K)
                    tma_load_4d(tx, full + s, b_dst + q * L::ATOM, at_c[q], w + at_j[q] - a.pw, ho + at_i[q] - a.ph, n);
                else   // column atom beyond kh*kw*C: keep the transaction count with an all-out-of-bounds box
                    tma_load_4d(tx, full + s, b_dst + q * L::ATOM, 0, -256, 0, n);
            }
            if (++wb == sg.w_blocks) { wb = 0; if (++ho == a.Ho) { ho = 0; n += sg.bn; } }
        }
    }
}

template <int RB>
__global__ void __launch_bounds__(kPpThreads, 1)
conv_wgrad_pp_kernel(const __grid_constant__ WgradMaps tm, float *__restrict__ dW, const __grid_constant__ PpWgradArgs a) {
    using L = PpWgradSmem<RB>;
    constexpr int STAGES = L::STAGES;
    extern __shared__ unsigned char smem_raw[];
    unsigned char *smem = (unsigned char *)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint64_t *full = (uint64_t *)(smem + L::BAR_OFF);
    uint64_t *empty = full + STAGES;
    const int wg = threadIdx.x >> 7;

    if (threadIdx.x == 0) {
        for (int q = 0; q < a.nseg; ++q) { tma_prefetch_desc(&tm.dz[q]); tma_prefetch_desc(&tm.x[q]); }
        for (int s = 0; s < STAGES; ++s) { mbar_init(full + s, 1); mbar_init(empty + s, 2); }   // empty: both consumers
        fence_barrier_init();
    }
    __syncthreads();

    if (wg == 0) {
        // ------------------------------------------------------------ producer
        reg_dec<kPpProducerRegs>();
        if (threadIdx.x < 32 && elect_one()) wgrad_produce<L, 4>(tm, a, smem, full, empty);
        return;
    }

    // ---------------------------------------------------------------- consumers: column half c of every tile
    reg_inc<kPpConsumerRegs>();
    const int c = wg - 1;
    const int mt_ = threadIdx.x & 127;
    const int w = mt_ >> 5, l = mt_ & 31;
    const bool odd = l & 1;
    uint32_t it = 0;
    for (int u = blockIdx.x; u < a.units; u += gridDim.x) {
        const WgradUnit un = wgrad_unit(a, u);
        const int tile = un.tile, nkb = un.kb_hi - un.kb_lo;
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

// =====================================================================================================
// The same weight gradient with 128 (Cout) x 192 (kh*kw*C columns) tiles, for K = 576 and 1152 (L1 and L2 of the CRNN),
// which 256-column tiles cover only with 768 and 1280 columns.  The producer, segment plan and split schedule are those of
// conv_wgrad_pp_kernel; a stage holds the two 64-row dz atoms and three 64-column x atoms.  Both consumers read the whole
// x stage and consumer c multiplies dz atom c (Cout rows 64c..64c+63) by it, one m64n192k16 per 16-deep step.
// =====================================================================================================
template <int RB> struct N192WgradSmem {
    static constexpr int STAGES = RB == 64 ? 5 : 4;
    static constexpr int ATOM = RB * 128;
    static constexpr int A_BYTES = 2 * ATOM;               // 128 output channels
    static constexpr int B_BYTES = 3 * ATOM;               // 192 columns
    static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
    static constexpr int BAR_OFF = STAGES * STAGE_BYTES;
    static constexpr int TOTAL = BAR_OFF + 2 * STAGES * 8 + 1024;
    static_assert(TOTAL <= 232448, "227 KB of opt-in shared memory");
};

template <int RB>
__global__ void __launch_bounds__(kPpThreads, 1)
conv_wgrad_n192_kernel(const __grid_constant__ WgradMaps tm, float *__restrict__ dW, const __grid_constant__ PpWgradArgs a) {
    using L = N192WgradSmem<RB>;
    constexpr int STAGES = L::STAGES;
    extern __shared__ unsigned char smem_raw[];
    unsigned char *smem = (unsigned char *)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint64_t *full = (uint64_t *)(smem + L::BAR_OFF);
    uint64_t *empty = full + STAGES;
    const int wg = threadIdx.x >> 7;

    if (threadIdx.x == 0) {
        for (int q = 0; q < a.nseg; ++q) { tma_prefetch_desc(&tm.dz[q]); tma_prefetch_desc(&tm.x[q]); }
        for (int s = 0; s < STAGES; ++s) { mbar_init(full + s, 1); mbar_init(empty + s, 2); }   // empty: both consumers
        fence_barrier_init();
    }
    __syncthreads();

    if (wg == 0) {
        reg_dec<kPpProducerRegs>();
        if (threadIdx.x < 32 && elect_one()) wgrad_produce<L, 3>(tm, a, smem, full, empty);
        return;
    }

    // ---------------------------------------------------------------- consumers: row half c of every tile
    reg_inc<kPpConsumerRegs>();
    const int c = wg - 1;
    const int mt_ = threadIdx.x & 127;
    const int w = mt_ >> 5, l = mt_ & 31;
    const bool odd = l & 1;
    uint32_t it = 0;
    for (int u = blockIdx.x; u < a.units; u += gridDim.x) {
        const WgradUnit un = wgrad_unit(a, u);
        const int tile = un.tile, nkb = un.kb_hi - un.kb_lo;
        if (nkb == 0) continue;
        const int mt = tile / a.n_tiles;
        const int m0 = mt * BM + c * 64, n0 = (tile - mt * a.n_tiles) * 192;
        float d[96];
        // not unrolled: a peeled first block makes ptxas copy the accumulator between in-flight wgmmas (C7514)
#pragma unroll 1
        for (int i = 0; i < nkb; ++i, ++it) {
            const int s = it % STAGES;
            mbar_wait(full + s, (it / STAGES) & 1);
            wgmma_fence();
            const uint32_t a_addr = smem_u32(smem + s * L::STAGE_BYTES);
            const uint32_t b_addr = a_addr + L::A_BYTES;
#pragma unroll
            for (int k = 0; k < RB / WGMMA_K; ++k)
                Wgmma<192>::template mma<1, 1>(d, desc_mnmajor(a_addr, k, L::ATOM, c), desc_mnmajor(b_addr, k, L::ATOM),
                                               (i | k) != 0);
            wgmma_commit();
            wgmma_wait<1>();
            if (i > 0 && mt_ == 0) mbar_arrive(empty + (it - 1) % STAGES);
        }
        wgmma_wait<0>();
        if (mt_ == 0) mbar_arrive(empty + (it - 1) % STAGES);
        // Fragment d[4j + 2h + e] is row 16 w + l / 4 + 8 h, column 8 j + 2 (l % 4) + e; the pair swap of
        // conv_wgrad_pp_kernel's flush gives each lane 4 consecutive columns of one row.
        const int col0 = n0 + 2 * (l & 3) - (odd ? 2 : 0);
        const int row = m0 + 16 * w + (l >> 2) + (odd ? 8 : 0);
        float *dst = dW + (int64_t)row * a.K + col0;
#pragma unroll
        for (int j = 0; j < 24; ++j) {
            const float *q = &d[4 * j];
            const float r0 = __shfl_xor_sync(0xffffffffu, odd ? q[0] : q[2], 1);
            const float r1 = __shfl_xor_sync(0xffffffffu, odd ? q[1] : q[3], 1);
            if (row < a.Cout && col0 + 8 * j < a.K) {
                if (odd) red_add_v4(dst + 8 * j, r0, r1, q[2], q[3]);
                else red_add_v4(dst + 8 * j, q[0], q[1], r0, r1);
            }
        }
    }
}

template <int BN>
int launch_pp(const CUtensorMap &tb, const CUtensorMap *tx, const CUtensorMap *ty, const PpConvArgs &a, int grid,
              cudaStream_t st) {
    auto kern = conv_fprop_pp_kernel<BN>;
    constexpr int smem = PpSmem<BN>::TOTAL > PpHaloSmem<BN>::TOTAL ? PpSmem<BN>::TOTAL : PpHaloSmem<BN>::TOTAL;
    { int rc = ensure_dyn_smem((const void *)kern, smem, "conv_fprop_pp smem attr"); if (rc) return rc; }
    kern<<<grid, kPpThreads, smem, st>>>(tb, tx[0], tx[1], tx[2], tx[3], ty[0], ty[1], ty[2], ty[3], a);
    return check_launch("conv_fprop_pp_kernel");
}

template <int BN>
int launch_m256(const CUtensorMap &tb, const CUtensorMap *tx, const CUtensorMap *ty, const PpConvArgs &a, int grid,
                cudaStream_t st) {
    auto kern = conv_fprop_m256_kernel<BN>;
    { int rc = ensure_dyn_smem((const void *)kern, M256Smem<BN>::TOTAL, "conv_fprop_m256 smem attr"); if (rc) return rc; }
    kern<<<grid, kPpThreads, M256Smem<BN>::TOTAL, st>>>(tb, tx[0], tx[1], tx[2], tx[3], ty[0], ty[1], ty[2], ty[3], a);
    return check_launch("conv_fprop_m256_kernel");
}

template <int RB>
int launch_wgrad_pp(const WgradMaps &tm, float *dW, const PpWgradArgs &a, int grid, cudaStream_t st) {
    auto kern = conv_wgrad_pp_kernel<RB>;
    { int rc = ensure_dyn_smem((const void *)kern, PpWgradSmem<RB>::TOTAL, "conv_wgrad_pp smem attr"); if (rc) return rc; }
    kern<<<grid, kPpThreads, PpWgradSmem<RB>::TOTAL, st>>>(tm, dW, a);
    return check_launch("conv_wgrad_pp_kernel");
}

template <int RB>
int launch_wgrad_n192(const WgradMaps &tm, float *dW, const PpWgradArgs &a, int grid, cudaStream_t st) {
    auto kern = conv_wgrad_n192_kernel<RB>;
    { int rc = ensure_dyn_smem((const void *)kern, N192WgradSmem<RB>::TOTAL, "conv_wgrad_n192 smem attr"); if (rc) return rc; }
    kern<<<grid, kPpThreads, N192WgradSmem<RB>::TOTAL, st>>>(tm, dW, a);
    return check_launch("conv_wgrad_n192_kernel");
}

// The weight gradient's schedule on at most `ctas` (>= 1) CTAs with 128 x tile_n tiles: segments, tiles, splits and grid.
// *balanced: every CTA gets the same number of units.
int plan_wgrad(int N, int Ho, int Wo, int C, int Cout, int kh, int kw, int ph, int pw, int ctas, int min_kb, int tile_n,
               PpWgradArgs *pa, int *grid_out, bool *balanced) {
    PpWgradArgs &a = *pa;
    a.C = C; a.Cout = Cout; a.K = kh * kw * C; a.kw = kw; a.ph = ph; a.pw = pw; a.Ho = Ho;
    const int64_t kb_total = plan_wgrad_segments(N, Ho, Wo, wgrad_rb(Wo), a.seg, &a.nseg);
    a.n_tiles = (int)ceil_div(a.K, tile_n);
    const int64_t tiles = ceil_div(Cout, BM) * a.n_tiles;
    if (kb_total * tiles > (1LL << 31) / 2) return MR_ERR_UNSUPPORTED;
    a.kb_total = (int)kb_total;
    a.tiles = (int)tiles;
    if (ctas > kb_total * tiles) ctas = (int)(kb_total * tiles);
    if (min_kb < 1) min_kb = 1;
    /* The plan makes splits x tiles a whole multiple of the grid, and lets the grid go down to 90 % of `ctas` for it:
     * (1) one unit per CTA, splits = ctas / tiles, when that fills 90 % of the CTAs;
     * (2) otherwise the largest such grid g whose fewest splits, g / gcd(g, tiles), keep min_kb K blocks each;
     * (3) otherwise (few K blocks, or few CTAs) ctas / tiles splits, as many as min_kb allows, and some CTAs get one unit
     *     more than others. */
    int64_t splits = std::min<int64_t>(kb_total, std::max<int64_t>(1, ctas / tiles));
    int64_t grid = 0;
    if (splits * tiles <= ctas && splits * tiles * 10 >= (int64_t)ctas * 9) grid = splits * tiles;
    for (int g = ctas; grid == 0 && (int64_t)g * 10 >= (int64_t)ctas * 9; --g) {
        const int64_t s = g / std::gcd<int64_t>(g, tiles);
        if (kb_total >= s * min_kb) { splits = s; grid = g; }
    }
    *balanced = grid != 0;
    if (grid == 0) {
        splits = std::max<int64_t>(1, std::min<int64_t>(splits, kb_total / min_kb));
        grid = std::min<int64_t>(ctas, splits * tiles);
    }
    a.kb_split = (int)ceil_div(kb_total, splits);
    a.units = (int)(splits * tiles);
    *grid_out = (int)grid;
    return MR_OK;
}

// Halo mode (pp_halo) for a call of conv_fprop_pp_kernel: every pixel tile one whole 128-pixel output row, kw > 1 taps
// sharing it, and at most kHaloSlots channel blocks.  The row geometry does not depend on N.
bool pp_halo_mode(int Wo, int C, int kw, const ConvSeg *seg, int nseg) {
    if (kw < 2 || kw > kHaloMaxKw || C / BK > kHaloSlots || nseg == 0) return false;
    for (int q = 0; q < nseg; ++q)
        if (seg[q].bw != 128 || seg[q].bh != 1 || seg[q].bn != 1) return false;
    return Wo % 128 == 0;
}

// The weight-gradient entries: mr_conv_wgrad_pp (tile_n = 256, conv_wgrad_pp_kernel) and mr_conv_wgrad_n192 (tile_n = 192,
// conv_wgrad_n192_kernel) differ only in the tile width.
int wgrad_entry(int tile_n, const void *dz, const void *x, float *dWm, int N, int H, int W, int C, int Cout, int kh, int kw,
                int ph, int pw, int ctas, int min_kb, void *stream) {
    if (N < 0 || H <= 0 || W <= 0 || C <= 0 || Cout <= 0 || kh <= 0 || kw <= 0 || ph < 0 || pw < 0) return MR_ERR_BAD_SHAPE;
    const int Ho = H + 2 * ph - kh + 1, Wo = W + 2 * pw - kw + 1;
    if (Ho <= 0 || Wo <= 0) return MR_ERR_BAD_SHAPE;
    if (N == 0) return MR_OK;
    if (!dz || !x || !dWm) return MR_ERR_NULL_POINTER;
    if (C % 64 || Cout % 8 || ((uintptr_t)x % 16) || ((uintptr_t)dz % 16) || ((uintptr_t)dWm % 16)) return MR_ERR_UNSUPPORTED;
    const int sms = sm_count();
    if (sms <= 0) { set_cuda_error(cudaErrorUnknown, "multiprocessor count"); return MR_ERR_CUDA; }
    if (ctas <= 0 || ctas > sms) ctas = sms;
    PpWgradArgs a;
    int grid = 0;
    bool balanced = false;
    int rc = plan_wgrad(N, Ho, Wo, C, Cout, kh, kw, ph, pw, ctas, min_kb, tile_n, &a, &grid, &balanced);
    if (rc) return rc;
    WgradMaps tm;
    for (int q = 0; q < kMaxWgradSegs; ++q) {
        const WgradSeg &s = a.seg[q < a.nseg ? q : 0];
        rc = make_map_nhwc(&tm.dz[q], dz, Cout, Wo, Ho, N, s.bw, 1, s.bn);
        if (rc) return rc;
        rc = make_map_nhwc(&tm.x[q], x, C, W, H, N, s.bw, 1, s.bn);
        if (rc) return rc;
    }
    cudaStream_t st = (cudaStream_t)stream;
    const bool rb80 = wgrad_rb(Wo) == 80;
    if (tile_n == 192)
        return rb80 ? launch_wgrad_n192<80>(tm, dWm, a, grid, st) : launch_wgrad_n192<64>(tm, dWm, a, grid, st);
    return rb80 ? launch_wgrad_pp<80>(tm, dWm, a, grid, st) : launch_wgrad_pp<64>(tm, dWm, a, grid, st);
}

int wgrad_plan_entry(int tile_n, int N, int H, int W, int C, int Cout, int kh, int kw, int ph, int pw, int ctas, int min_kb,
                     int *plan) {
    if (N <= 0 || H <= 0 || W <= 0 || C <= 0 || Cout <= 0 || kh <= 0 || kw <= 0 || ph < 0 || pw < 0 || ctas <= 0)
        return MR_ERR_BAD_SHAPE;
    const int Ho = H + 2 * ph - kh + 1, Wo = W + 2 * pw - kw + 1;
    if (Ho <= 0 || Wo <= 0) return MR_ERR_BAD_SHAPE;
    if (!plan) return MR_ERR_NULL_POINTER;
    PpWgradArgs a;
    int grid = 0;
    bool balanced = false;
    const int rc = plan_wgrad(N, Ho, Wo, C, Cout, kh, kw, ph, pw, ctas, min_kb, tile_n, &a, &grid, &balanced);
    if (rc) return rc;
    int *p = plan;
    *p++ = wgrad_rb(Wo); *p++ = grid; *p++ = a.kb_total; *p++ = a.tiles; *p++ = a.kb_split; *p++ = a.units;
    *p++ = balanced; *p++ = a.nseg;
    for (int q = 0; q < kMaxWgradSegs; ++q) {
        const WgradSeg s = q < a.nseg ? a.seg[q] : WgradSeg{0, 0, 0, 0, 0};
        *p++ = s.w0; *p++ = s.bw; *p++ = s.bn; *p++ = s.w_blocks; *p++ = s.kb_begin;
    }
    return MR_OK;
}

}  // namespace

extern "C" {

/* Persistent implicit-GEMM stride-1 convolution on NHWC bf16: y[N*Ho*Wo, Cout] bf16 = conv(x[N,H,W,C], Wm[Cout, kh*kw*C]);
 * no bias, no activation.  With flipped/transposed weights and padding (k-1-p) it is the input gradient.  Wm's rows are
 * ldw elements apart (0: kh*kw*C), and y's images y_nstride elements apart (0: Ho*Wo*Cout), so a call can read a column
 * slice of a wider weight matrix and write rows of a taller output.  tile_m picks the kernel: 128 conv_fprop_pp_kernel,
 * 256 conv_fprop_m256_kernel (Cout > 64 only), 0 the faster one for the call, by its K-block count.  Bit-identical to
 * mr_conv_fprop_tcgen05 with a bf16 output whichever runs.  MR_ERR_UNSUPPORTED unless C % 64 == 0, Cout % 8 == 0, the
 * pointers are 16-byte aligned, the strides are multiples of 8 elements and the output tiles with at most four TMA box
 * segments. */
int mr_conv_fprop_pp(const void *x, const void *Wm, void *y, int N, int H, int W, int C, int Cout, int kh, int kw, int ph,
                     int pw, int ldw, int y_nstride, int tile_m, void *stream) {
    if (N < 0 || H <= 0 || W <= 0 || C <= 0 || Cout <= 0 || kh <= 0 || kw <= 0 || ph < 0 || pw < 0) return MR_ERR_BAD_SHAPE;
    const int Ho = H + 2 * ph - kh + 1, Wo = W + 2 * pw - kw + 1;
    if (Ho <= 0 || Wo <= 0) return MR_ERR_BAD_SHAPE;
    const int64_t K = (int64_t)kh * kw * C;
    if (ldw == 0) ldw = (int)K;
    if (ldw < K || (y_nstride != 0 && y_nstride < (int64_t)Ho * Wo * Cout)) return MR_ERR_BAD_SHAPE;
    if (tile_m != 0 && tile_m != 128 && tile_m != 256) return MR_ERR_BAD_SHAPE;
    if (N == 0) return MR_OK;
    if (!x || !Wm || !y) return MR_ERR_NULL_POINTER;
    if (C % 64 || Cout % 8 || ((uintptr_t)x % 16) || ((uintptr_t)Wm % 16) || ((uintptr_t)y % 16)) return MR_ERR_UNSUPPORTED;
    if (ldw % 8 || y_nstride % 8) return MR_ERR_UNSUPPORTED;
    if ((int64_t)N * Ho * Wo > (1LL << 31) - 256) return MR_ERR_UNSUPPORTED;
    const int BN = Cout > 64 ? 128 : 64;
    const bool m256 = tile_m == 256 || (tile_m == 0 && K / BK >= kM256MinKb);
    if (m256 && BN != 128) return MR_ERR_UNSUPPORTED;
    PpConvArgs a;
    a.C = C; a.Cout = Cout; a.kh = kh; a.kw = kw; a.ph = ph; a.pw = pw;
    CUtensorMap tx[kMaxConvSegs], ty[kMaxConvSegs];
    int pixel_tiles = 0;
    int rc = plan_conv_segments(x, N, H, W, C, Ho, Wo, 1, 1, a.seg, tx, &a.nseg, &pixel_tiles);
    if (rc) return rc;
    if (a.nseg == 0) return MR_ERR_UNSUPPORTED;
    for (int q = 0; q < a.nseg; ++q) {
        rc = make_map_nhwc(&ty[q], y, Cout, Wo, Ho, N, a.seg[q].bw, a.seg[q].bh, a.seg[q].bn, 1, 1, y_nstride);
        if (rc) return rc;
    }
    for (int q = a.nseg; q < kMaxConvSegs; ++q) { tx[q] = tx[0]; ty[q] = ty[0]; }
    CUtensorMap tb;
    rc = make_map(&tb, Wm, K, Cout, ldw, BK, BN);
    if (rc) return rc;
    a.halo = !m256 && pp_halo_mode(Wo, C, kw, a.seg, a.nseg);
    if (a.halo) {                                              // one map for every segment: the box is a whole halo row
        rc = make_map_nhwc(&tx[0], x, C, W, H, N, 128 + kw - 1, 1, 1);
        if (rc) return rc;
    }
    a.pix_tiles = pixel_tiles;
    a.cout_tiles = (int)ceil_div(Cout, BN);
    const int64_t tiles = (m256 ? ceil_div(pixel_tiles, 2) : (int64_t)pixel_tiles) * a.cout_tiles;
    if (tiles > (1LL << 31) - 1) return MR_ERR_UNSUPPORTED;
    a.tiles = (int)tiles;
    const int sms = sm_count();
    if (sms <= 0) { set_cuda_error(cudaErrorUnknown, "multiprocessor count"); return MR_ERR_CUDA; }
    const int grid = (int)(tiles < sms ? tiles : sms);
    cudaStream_t st = (cudaStream_t)stream;
    if (m256) return launch_m256<128>(tb, tx, ty, a, grid, st);
    return BN == 128 ? launch_pp<128>(tb, tx, ty, a, grid, st) : launch_pp<64>(tb, tx, ty, a, grid, st);
}

/* Host only: 1 when mr_conv_fprop_pp runs this geometry with tile_m = 0 in conv_fprop_pp_kernel's halo mode (one activation
 * halo per tap row and channel block, shared by the row's kw taps), 0 when it does not, MR_ERR_BAD_SHAPE for an invalid
 * geometry.  The halo mode
 * needs output rows of whole 128-pixel tiles (Wo a multiple of 128, at most four of them), 2 <= kw <= 8 and C <= 256. */
int mr_conv_fprop_pp_halo(int H, int W, int C, int Cout, int kh, int kw, int ph, int pw) {
    if (H <= 0 || W <= 0 || C <= 0 || Cout <= 0 || kh <= 0 || kw <= 0 || ph < 0 || pw < 0) return MR_ERR_BAD_SHAPE;
    const int Ho = H + 2 * ph - kh + 1, Wo = W + 2 * pw - kw + 1;
    if (Ho <= 0 || Wo <= 0) return MR_ERR_BAD_SHAPE;
    if (C % BK || (int64_t)kh * kw * C / BK >= kM256MinKb) return 0;   // refused, or the 256-pixel kernel's call
    ConvSeg seg[kMaxConvSegs];
    int nseg = 0;
    for (int w0 = 0; w0 < Wo; w0 += 128) {                     // plan_conv_segments' widths, without the tensor maps
        if (Wo - w0 < 128 || nseg == kMaxConvSegs) return 0;
        seg[nseg++] = ConvSeg{w0, 128, 1, 1, Ho, 0};
    }
    return pp_halo_mode(Wo, C, kw, seg, nseg) ? 1 : 0;
}

/* Persistent implicit-GEMM weight gradient, stride 1: dWm[Cout, kh*kw*C] fp32 (ACCUMULATED atomically: zero it first) from
 * dz[N,Ho,Wo,Cout] and x[N,H,W,C] (NHWC bf16) on at most `ctas` CTAs (<= 0 or more than the SMs: one per SM), with at least
 * `min_kb` K blocks per split where the plan allows it.  MR_ERR_UNSUPPORTED unless C % 64 == 0, Cout % 8 == 0 and 16-byte
 * aligned operands. */
int mr_conv_wgrad_pp(const void *dz, const void *x, float *dWm, int N, int H, int W, int C, int Cout, int kh, int kw, int ph,
                     int pw, int ctas, int min_kb, void *stream) {
    return wgrad_entry(256, dz, x, dWm, N, H, W, C, Cout, kh, kw, ph, pw, ctas, min_kb, stream);
}

/* mr_conv_wgrad_pp with 128 x 192 tiles (conv_wgrad_n192_kernel): no idle column atoms where kh*kw*C is a multiple of 192
 * but not of 256. */
int mr_conv_wgrad_n192(const void *dz, const void *x, float *dWm, int N, int H, int W, int C, int Cout, int kh, int kw, int ph,
                       int pw, int ctas, int min_kb, void *stream) {
    return wgrad_entry(192, dz, x, dWm, N, H, W, C, Cout, kh, kw, ph, pw, ctas, min_kb, stream);
}

/* Host only: the schedule mr_conv_wgrad_pp runs on `ctas` (>= 1) CTAs, into plan[MR_WGRAD_PP_PLAN_INTS]:
 * {RB, grid, kb_total, tiles, kb_split, units, balanced, nseg, then nseg x (w0, bw, bn, w_blocks, kb_begin)}. */
int mr_conv_wgrad_pp_plan(int N, int H, int W, int C, int Cout, int kh, int kw, int ph, int pw, int ctas, int min_kb,
                          int *plan) {
    return wgrad_plan_entry(256, N, H, W, C, Cout, kh, kw, ph, pw, ctas, min_kb, plan);
}

/* Host only: the same for mr_conv_wgrad_n192 (tiles counts 128 x 192 tiles). */
int mr_conv_wgrad_n192_plan(int N, int H, int W, int C, int Cout, int kh, int kw, int ph, int pw, int ctas, int min_kb,
                            int *plan) {
    return wgrad_plan_entry(192, N, H, W, C, Cout, kh, kw, ph, pw, ctas, min_kb, plan);
}

}  // extern "C"
