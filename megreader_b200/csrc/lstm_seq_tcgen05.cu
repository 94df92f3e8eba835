// Persistent bidirectional-LSTM recurrence for sm_90a (decoders/crnn.py:13,17 nn.LSTM inside BidirectionalLSTM).
//
// The recurrence h_t = cell(Gx_t + h_{t-1} W_hh^T) is T dependent steps of a small GEMM ([B,H] x [H,4H]) plus a
// transcendental-heavy cell.  Launched step by step it is launch- and latency-bound (2 launches x T x 2 layers x
// fwd/bwd = 520 short launches in the CRNN train step).  Here ONE launch runs the whole sequence of one layer,
// both directions:
//   * the CTA grid tiles batch rows x gate columns (fwd) / hidden units (bwd) x direction and stays resident for all T steps;
//   * each CTA keeps its W_hh slice in shared memory for the whole sequence (loaded once by TMA);
//   * per step one producer thread waits for the peers' arrivals and TMA-loads h_{t-1} (fwd) / dG_{t+1} (bwd), which
//     are L2-resident; each consumer warpgroup accumulates the recurrent product of its 64 rows with wgmma and applies
//     the cell to the accumulator fragments in its registers; the cell state (fwd) / its gradient (bwd) never leaves
//     registers;
//   * the CTAs that share batch rows exchange h_t (fwd) / dG_t (bwd) through global memory and a monotonically
//     increasing arrival counter per (direction, row tile): writers  st -> bar.sync (the warpgroup) -> red.release.gpu,
//     readers  ld.acquire spin -> fence.proxy.async -> TMA.  All CTAs must be co-resident: the host refuses grids
//     larger than the device can hold (MR_ERR_UNSUPPORTED -> callers use the per-step kernels).
// Gate columns are UNIT-MAJOR (column 4*j + g = gate g of hidden unit j; g = i,f,g,o) as in gemm_tcgen05.cu.
// Every wait is bounded: on timeout the CTA records an error word (the last word of flags) and runs to completion with
// undefined results instead of hanging the device.
#include "wgmma.cuh"
#include "lstm_cell.cuh"
#include <stdlib.h>

namespace {

constexpr int kBN = 64;                       // gate columns per forward CTA
constexpr int kSeqRows = 64;                  // batch rows per consumer warpgroup (one m64 wgmma row block)
constexpr int kFwdThreads = 3 * kMmaThreads;  // producer warpgroup + two consumer warpgroups (rows 0..63, 64..127)
constexpr int kFwdProducerRegs = 40;
constexpr int kFwdConsumerRegs = 232;
static_assert(kMmaThreads * kFwdProducerRegs + 2 * kMmaThreads * kFwdConsumerRegs <= 65536, "register file");

__device__ __forceinline__ uint32_t ld_acquire(const unsigned *p) {
    uint32_t v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
// Publishes every write that happens-before it (the warpgroup's stores, ordered by the preceding bar.sync) to a peer that
// acquires the counter: release semantics, without the full fence of __threadfence() + atomicAdd.
__device__ __forceinline__ void red_release_add(unsigned *p, unsigned v) {
    asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }

#define MR_TRACE(step, slot) do { if (trace) trace[(step) * 32 + (slot)] = clock64(); } while (0)
__device__ __forceinline__ uint64_t now_ns() { uint64_t t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); return t; }
constexpr uint64_t kTimeoutNs = 2000000000ull;     // 2 s: ~10^5 x the longest legitimate wait

// Bounded waits: give up (false) when the error word is already set or after kTimeoutNs, so that a protocol failure
// drains the grid in bounded time instead of hanging the device.
__device__ __forceinline__ bool mbar_wait_bounded(uint64_t *bar, uint32_t parity, const volatile unsigned *err) {
    uint64_t t0 = 0;
    for (uint32_t it = 1;; ++it) {
        uint32_t ok;
        asm volatile(
            "{\n"
            ".reg .pred p;\n"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
            "selp.u32 %0, 1, 0, p;\n"
            "}\n" : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
        if (ok) return true;
        if ((it & 63u) == 0) {
            if (*err) return false;
            const uint64_t t = now_ns();
            if (!t0) t0 = t;
            else if (t - t0 > kTimeoutNs) return false;
        }
    }
}
__device__ __forceinline__ bool flag_wait_bounded(const unsigned *flag, uint32_t target, const volatile unsigned *err) {
    uint64_t t0 = 0;
    for (uint32_t it = 1;; ++it) {
        if (ld_acquire(flag) >= target) return true;
        if ((it & 63u) == 0) {
            if (*err) return false;
            const uint64_t t = now_ns();
            if (!t0) t0 = t;
            else if (t - t0 > kTimeoutNs) return false;
        }
    }
}

__device__ __forceinline__ void tma_load_3d(const CUtensorMap *map, uint64_t *bar, void *dst, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
                 ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void tma_store_3d(const CUtensorMap *map, const void *src, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
                 ::"l"(map), "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void tma_store_commit_wait_read() {      // until the stores have READ their smem source
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}
// 16-byte chunk `c` of row `r` in a [rows x 128 B] tile written by TMA with the 128-byte swizzle (tile base 1024-aligned)
__device__ __forceinline__ uint32_t swz(int r, int c) { return (uint32_t)(r * 128 + ((c ^ (r & 7)) << 4)); }
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
    const __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<const uint32_t *>(&v);
}

// Accumulator fragment of wgmma m64nNk16 (AccTile): thread mt of the warpgroup (warp w = mt / 32, lane l) holds rows
// 16 w + l / 4 and 16 w + l / 4 + 8 (h = 0, 1) at columns 8 j + 2 (l % 4) + e, as d[4 j + 2 h + e].

struct SeqFwdArgs {
    bf16 *G;                  // [2, T, B, 4H] unit-major: x-projection on entry, activated gates on exit
    const float *bias[2];     // [4H] unit-major, b_ih + b_hh
    float *C;                 // [2, T, B, H] cell states (saved for the backward pass)
    bf16 *Y;                  // [T, B, 2H] layer output: direction d owns columns [d*H, (d+1)*H)
    unsigned *flags;          // [2 * ceil(B / 64) + 1], zeroed before launch: counters [dir][row tile], last word = error
    unsigned *err;            // the error word
    long long *trace;         // optional [T][32] clock64 stamps of CTA (0,0,0) (mr_lstm_seq_set_trace), else NULL
    int T, B, H;
};

// Forward: a CTA owns 128 batch rows x 64 gate columns (16 hidden units).  Consumer warpgroup c issues the wgmma
// m64n64k16 sequence of rows 64c..64c+63 (the per-step kernels' K order) and keeps the fragment in registers.  A
// fragment column pair is (i, f) or (g, o) of one unit (unit-major columns), so lanes 2k and 2k + 1 -- which hold the
// other pair of the same unit for the same two rows -- swap one row's pair: the even lane then applies the cell to row
// h = 0, the odd lane to row h = 1, eight units each (units 2 j + (l % 4) / 2 of the tile).  The x-projection and the
// cell-state output go through TMA-staged tiles of the warpgroup's 64 rows; each warpgroup posts its own arrival.
__global__ void __launch_bounds__(kFwdThreads, 1)
lstm_seq_fwd_kernel(const __grid_constant__ CUtensorMap tmY, const __grid_constant__ CUtensorMap tmW0,
                    const __grid_constant__ CUtensorMap tmW1, const __grid_constant__ CUtensorMap tmG3,
                    const __grid_constant__ CUtensorMap tmC3, SeqFwdArgs a) {
    extern __shared__ unsigned char smem_raw[];
    unsigned char *smem = (unsigned char *)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    const int nkb = a.H / BK;
    unsigned char *As = smem;                             // nkb x [128 rows x 128 B]   h_{t-1} tile, K-major SW128
    unsigned char *Ws = smem + nkb * 16384;               // nkb x [ 64 rows x 128 B]   W_hh slice, K-major SW128
    unsigned char *Gt = Ws + nkb * 8192;                  // [2 warpgroups][2 steps] x [64 rows x 128 B]   gates: x-projection in, activations out
    unsigned char *Ct = Gt + 32768;                       // [2 warpgroups] x [64 rows x 64 B]             cell states (16 units fp32), out
    uint64_t *wfull = (uint64_t *)(Ct + 8192);
    uint64_t *afull = wfull + 1;                          // [8]
    uint64_t *gfull = afull + 8;                          // [2 warpgroups][2 steps]

    const int dir = blockIdx.z;
    const CUtensorMap *tmW = dir ? &tmW1 : &tmW0;
    const int m0 = blockIdx.x * BM, n0 = blockIdx.y * kBN;
    const int T = a.T, B = a.B, H = a.H;
    unsigned *flag = a.flags + dir * gridDim.x + blockIdx.x;
    unsigned *err = a.err;
    const uint32_t arrivals = 2 * gridDim.y;              // per step: one per consumer warpgroup of every column tile
    long long *trace = (blockIdx.x | blockIdx.y | blockIdx.z) == 0 ? a.trace : nullptr;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmY);
        tma_prefetch_desc(tmW);
        tma_prefetch_desc(&tmG3);
        tma_prefetch_desc(&tmC3);
        mbar_init(wfull, 1);
        for (int i = 0; i < 8; ++i) mbar_init(afull + i, 1);
        for (int i = 0; i < 4; ++i) mbar_init(gfull + i, 1);
        fence_barrier_init();
    }
    __syncthreads();

    if (threadIdx.x < kMmaThreads) {
        reg_dec<kFwdProducerRegs>();
        if (threadIdx.x < 32 && elect_one()) {
            mbar_expect_tx(wfull, nkb * 8192);
            for (int kb = 0; kb < nkb; ++kb) tma_load_2d(tmW, wfull, Ws + kb * 8192, kb * BK, n0);
            for (int s = 1; s < T; ++s) {
                const int t_prev = dir ? T - s : s - 1;
                if (!flag_wait_bounded(flag, arrivals * (uint32_t)s, err)) atomicExch(err, 1u);
                MR_TRACE(s, 0);
                fence_proxy_async_global();
                for (int kb = 0; kb < nkb; ++kb) {
                    mbar_expect_tx(afull + kb, 16384);
                    tma_load_2d(&tmY, afull + kb, As + kb * 16384, dir * H + kb * BK, t_prev * B + m0);
                }
                MR_TRACE(s, 1);
            }
        }
        return;
    }

    reg_inc<kFwdConsumerRegs>();
    const int c = (threadIdx.x >> 7) - 1;                 // consumer warpgroup: rows 64c..64c+63 of the tile
    const int mt = threadIdx.x & 127, w = mt >> 5, l = mt & 31;
    const int hsel = l & 1;                               // fragment row this lane applies the cell to; also its gate pair: 0 (i, f), 1 (g, o)
    const int upar = (l >> 1) & 1;                        // units 2 j + upar of the tile, j = 0..7
    const int rl = 16 * w + (l >> 2) + 8 * hsel;          // row within the warpgroup's 64
    const int r0 = m0 + kSeqRows * c, row = r0 + rl;
    const bool live = row < B;
    const bool leader = mt == 0;
    if (!(leader && c == 0)) trace = nullptr;
    uint64_t *gf = gfull + 2 * c;
    unsigned char *gt0 = Gt + c * 16384, *ct = Ct + c * 4096;
    float bb[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const float4 b4 = __ldg(reinterpret_cast<const float4 *>((dir ? a.bias[1] : a.bias[0]) + n0 + 4 * (2 * j + upar)));
        bb[j][0] = b4.x; bb[j][1] = b4.y; bb[j][2] = b4.z; bb[j][3] = b4.w;
    }
    float cst[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) cst[j] = 0.f;
    auto time_of = [&](int s) { return dir ? T - 1 - s : s; };
    auto load_gates = [&](int s) {
        mbar_expect_tx(gf + (s & 1), 8192);
        tma_load_3d(&tmG3, gf + (s & 1), gt0 + (s & 1) * 8192, n0, r0, dir * T + time_of(s));
    };
    if (leader) {
        load_gates(0);
        if (T > 1) load_gates(1);
    }
    // The recurrent product of the step; each step's first wgmma overwrites it (scale-d = 0).  At s = 0 (no h_{-1}) it is
    // not read but replaced by zeros below: writing zeros into it would make ptxas serialize the wgmma.
    float acc[32];
    for (int s = 0; s < T; ++s) {
        const int t = time_of(s);
        unsigned char *gt = gt0 + (s & 1) * 8192;
        if (!mbar_wait_bounded(gf + (s & 1), (s >> 1) & 1, err)) atomicExch(err, 6u);
        uint2 px[8];                                      // x-projection (i, f, g, o) of this lane's 8 units
#pragma unroll
        for (int j = 0; j < 8; ++j) px[j] = *reinterpret_cast<const uint2 *>(gt + swz(rl, j) + 8 * upar);
        if (s > 0) {
            if (s == 1 && !mbar_wait_bounded(wfull, 0, err)) atomicExch(err, 2u);
            for (int kb = 0; kb < nkb; ++kb) {
                if (!mbar_wait_bounded(afull + kb, (s - 1) & 1, err)) atomicExch(err, 3u);
                const uint32_t a_addr = smem_u32(As + kb * 16384), b_addr = smem_u32(Ws + kb * 8192);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < BK / WGMMA_K; ++k)
                    Wgmma<kBN>::mma<0, 0>(acc, desc_kmajor(a_addr, k, c), desc_kmajor(b_addr, k), (kb | k) != 0);
                wgmma_commit();
            }
            MR_TRACE(s, 2);
            wgmma_wait<0>();
        }
        MR_TRACE(s, 3);
        float act[8][4], hn[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float own0 = hsel ? acc[4 * j + 2] : acc[4 * j], own1 = hsel ? acc[4 * j + 3] : acc[4 * j + 1];
            const float snd0 = hsel ? acc[4 * j] : acc[4 * j + 2], snd1 = hsel ? acc[4 * j + 1] : acc[4 * j + 3];
            const float rcv0 = __shfl_xor_sync(0xffffffffu, snd0, 1), rcv1 = __shfl_xor_sync(0xffffffffu, snd1, 1);
            float r[4] = {hsel ? rcv0 : own0, hsel ? rcv1 : own1, hsel ? own0 : rcv0, hsel ? own1 : rcv1};
#pragma unroll
            for (int g = 0; g < 4; ++g) r[g] = s > 0 ? r[g] : 0.f;
            const __nv_bfloat162 *x2 = reinterpret_cast<const __nv_bfloat162 *>(&px[j]);
            const float2 xa = __bfloat1622float2(x2[0]), xb = __bfloat1622float2(x2[1]);
            // rows >= B run on whatever their tiles hold: only their stores are skipped (h_t) or clipped (TMA)
            const LstmUnit u = lstm_unit_fwd<CellFast>(xa.x + r[0] + bb[j][0], xa.y + r[1] + bb[j][1],
                                                       xb.x + r[2] + bb[j][2], xb.y + r[3] + bb[j][3], cst[j]);
            cst[j] = u.c;
            hn[j] = u.h;
            act[j][0] = u.i; act[j][1] = u.f; act[j][2] = u.g; act[j][3] = u.o;
        }
        // Lanes l and l ^ 2 hold the even and the odd units of the same row: after swapping half of them each has eight
        // consecutive units (8 upar..8 upar + 7) of h_t and c_t for one 16-byte / two 16-byte stores.
        float hs[8], cs8[8];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float hr = __shfl_xor_sync(0xffffffffu, upar ? hn[k] : hn[4 + k], 2);
            const float cr = __shfl_xor_sync(0xffffffffu, upar ? cst[k] : cst[4 + k], 2);
            hs[2 * k] = upar ? hr : hn[k];          hs[2 * k + 1] = upar ? hn[4 + k] : hr;
            cs8[2 * k] = upar ? cr : cst[k];        cs8[2 * k + 1] = upar ? cst[4 + k] : cr;
        }
        if (live) {
            const uint4 hp = make_uint4(pack_bf16x2(hs[0], hs[1]), pack_bf16x2(hs[2], hs[3]), pack_bf16x2(hs[4], hs[5]),
                                        pack_bf16x2(hs[6], hs[7]));
            *reinterpret_cast<uint4 *>(a.Y + ((int64_t)t * B + row) * 2 * H + dir * H + (n0 >> 2) + 8 * upar) = hp;
        }
        // h_t is all the peers wait for: post the arrival before the state that only the backward pass reads
        MR_TRACE(s, 4);
        named_bar_sync<kMmaThreads>(1 + c);               // every h_t of the warpgroup's rows stored, As read by its wgmma
        MR_TRACE(s, 5);
        if (leader) {
            MR_TRACE(s, 6);
            red_release_add(flag, 1u);
            MR_TRACE(s, 7);
        }
        // activated gates back into the tile, cell state into its tile (rows >= B are clipped by the TMA store)
#pragma unroll
        for (int j = 0; j < 8; ++j)
            *reinterpret_cast<uint2 *>(gt + swz(rl, j) + 8 * upar) =
                make_uint2(pack_bf16x2(act[j][0], act[j][1]), pack_bf16x2(act[j][2], act[j][3]));
        *reinterpret_cast<float4 *>(ct + rl * 64 + 32 * upar) = make_float4(cs8[0], cs8[1], cs8[2], cs8[3]);   // plain rows
        *reinterpret_cast<float4 *>(ct + rl * 64 + 32 * upar + 16) = make_float4(cs8[4], cs8[5], cs8[6], cs8[7]);
        fence_proxy_async();                              // generic-proxy tile writes -> visible to the TMA stores
        named_bar_sync<kMmaThreads>(1 + c);
        if (leader) {
            const int z = dir * T + t;
            tma_store_3d(&tmG3, gt, n0, r0, z);
            tma_store_3d(&tmC3, ct, n0 >> 2, r0, z);
            tma_store_commit_wait_read();                 // both tiles may be overwritten again
            if (s + 2 < T) load_gates(s + 2);
        }
    }
    if (T == 1 && leader && !mbar_wait_bounded(wfull, 0, err)) atomicExch(err, 2u);   // no TMA load outlives the CTA
}

struct SeqBwdArgs {
    const bf16 *G;            // [2, T, B, 4H] activated gates (unit-major) from the forward pass
    const float *C;           // [2, T, B, H]
    const bf16 *dY;           // [T, B, 2H] gradient of the layer output
    bf16 *dG;                 // [2, T, B, 4H] gate gradients, out (unit-major)
    unsigned *flags;
    unsigned *err;
    long long *trace;
    int T, B, H;
};

// Backward recurrence: dh_{t} += dG_{t_next} W_hh needs the FULL gate-gradient row block [rows x 4H] per output tile, so
// the per-step operand traffic is (H / units-per-CTA) x the dG tile.  A CTA owns 64 batch rows x 32 hidden units:
// (B/64) x (H/32) x 2 CTAs (128 at the CRNN shape), each streaming a 64 x 4H dG row block per step through a ring that
// holds all of it at H = 256.  One consumer warpgroup issues the m64n32k16 sequence of the per-step kernels and applies
// the cell gradient to its fragment: lane l owns rows 16 w + l / 4 (+ 8) x units 8 j + 2 (l % 4) (+ 1), j = 0..3.  The
// activated gates [64 x 128] bf16 and cell states [64 x 32] fp32 of every step are TMA-loaded as swizzled tiles one step
// ahead and read conflict-free from shared memory; c_prev of this step is the c tile of the next one.
//
// dG_t leaves by plain 16-byte stores from registers.  Ordering: every consumer thread's stores precede the warpgroup's
// bar.sync, which precedes the leader's red.release.gpu (release is cumulative over what happens-before it); a peer's
// producer observes the count with ld.acquire.gpu, so the stores are visible to it, and its fence.proxy.async.global
// orders them before the async-proxy (TMA) reads of dG it issues next.
constexpr int kBwdBN = 32;
constexpr int kBwdWTile = kBwdBN * 128;       // one k-block of W_hh^T: 32 unit rows x 128 B (K-major, SW128)
constexpr int kBwdATile = kSeqRows * 128;     // one k-block of dG_{next}: 64 rows x 128 B
constexpr int kBwdThreads = kMmaThreads + 32; // the consumer warpgroup, then the producer warp

template <int STAGES>
__global__ void __launch_bounds__(kBwdThreads, 1)
lstm_seq_bwd_kernel(const __grid_constant__ CUtensorMap tmDG, const __grid_constant__ CUtensorMap tmW0,
                    const __grid_constant__ CUtensorMap tmW1, const __grid_constant__ CUtensorMap tmG3,
                    const __grid_constant__ CUtensorMap tmC3, SeqBwdArgs a) {
    extern __shared__ unsigned char smem_raw[];
    unsigned char *smem = (unsigned char *)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    const int nkb = 4 * a.H / BK;
    unsigned char *As = smem;                             // STAGES x [64 rows x 128 B]   dG_{next} k-block, K-major SW128
    unsigned char *Gs = smem + STAGES * kBwdATile;        // 2 x [64 x 128 B]             gates of this step (128 gate columns)
    unsigned char *Cs = Gs + 2 * kBwdATile;               // 2 x [64 x 128 B]             cell-state tiles (fp32, 32 units)
    unsigned char *Ws = Cs + 2 * kBwdATile;               // nkb x [32 rows x 128 B]      W_hh^T[n0.., kb*64..), K-major SW128
    uint64_t *wfull = (uint64_t *)(Ws + nkb * kBwdWTile);
    uint64_t *full = wfull + 1;
    uint64_t *empty = full + STAGES;
    uint64_t *gfull = empty + STAGES;
    uint64_t *cfull = gfull + 1;                          // [2]

    const int dir = blockIdx.z;
    const CUtensorMap *tmW = dir ? &tmW1 : &tmW0;
    const int m0 = blockIdx.x * kSeqRows, n0 = blockIdx.y * kBwdBN;
    const int T = a.T, B = a.B, H = a.H;
    unsigned *flag = a.flags + dir * gridDim.x + blockIdx.x;
    unsigned *err = a.err;
    const uint32_t arrivals = gridDim.y;
    long long *trace = (blockIdx.x | blockIdx.y | blockIdx.z) == 0 ? a.trace : nullptr;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmDG);
        tma_prefetch_desc(tmW);
        tma_prefetch_desc(&tmG3);
        tma_prefetch_desc(&tmC3);
        mbar_init(wfull, 1);
        for (int i = 0; i < STAGES; ++i) { mbar_init(full + i, 1); mbar_init(empty + i, 1); }
        mbar_init(gfull, 1);
        mbar_init(cfull, 1);
        mbar_init(cfull + 1, 1);
        fence_barrier_init();
    }
    __syncthreads();

    // processing order u = 0..T-1 is the reverse of the forward order: direction 0 walks t = T-1..0, direction 1 t = 0..T-1
    if (threadIdx.x >= kMmaThreads) {
        if (elect_one()) {
            mbar_expect_tx(wfull, nkb * kBwdWTile);
            for (int kb = 0; kb < nkb; ++kb) tma_load_2d(tmW, wfull, Ws + kb * kBwdWTile, kb * BK, n0);
            int it = 0;
            for (int u = 1; u < T; ++u) {
                const int t_next = dir ? u - 1 : T - u;          // the time index processed at order u-1
                if (!flag_wait_bounded(flag, arrivals * (uint32_t)u, err)) atomicExch(err, 1u);
                MR_TRACE(u, 0);
                fence_proxy_async_global();
                for (int kb = 0; kb < nkb; ++kb, ++it) {
                    const int s = it % STAGES;
                    if (!mbar_wait_bounded(empty + s, ((it / STAGES) & 1) ^ 1, err)) atomicExch(err, 5u);
                    mbar_expect_tx(full + s, kBwdATile);
                    if (kb >= 4 && kb < 12) MR_TRACE(u, 20 + kb);
                    tma_load_2d(&tmDG, full + s, As + s * kBwdATile, kb * BK, (dir * T + t_next) * B + m0);
                }
                MR_TRACE(u, 1);
            }
        }
        return;
    }

    const int mt = threadIdx.x, w = mt >> 5, l = mt & 31, q = l & 3;
    const bool leader = mt == 0;
    if (!leader) trace = nullptr;
    int rl[2], row[2];
    bool live[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        rl[h] = 16 * w + (l >> 2) + 8 * h;
        row[h] = m0 + rl[h];
        live[h] = row[h] < B;
    }
    float dcs[2][8];                                      // [h][2 j + e]: dL/dc of row h, unit 8 j + 2 q + e
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int k = 0; k < 8; ++k) dcs[h][k] = 0.f;
    auto time_of = [&](int u) { return dir ? u : T - 1 - u; };
    auto load_gates = [&](int u) {
        const int z = dir * T + time_of(u);
        mbar_expect_tx(gfull, 2 * kBwdATile);
        tma_load_3d(&tmG3, gfull, Gs, 4 * n0, m0, z);
        tma_load_3d(&tmG3, gfull, Gs + kBwdATile, 4 * n0 + 64, m0, z);
    };
    auto load_cell = [&](int u) {
        mbar_expect_tx(cfull + (u & 1), kBwdATile);
        tma_load_3d(&tmC3, cfull + (u & 1), Cs + (u & 1) * kBwdATile, n0, m0, dir * T + time_of(u));
    };
    if (leader) {
        load_gates(0);
        load_cell(0);
        if (T > 1) load_cell(1);
    }
    int it = 0;
    for (int u = 0; u < T; ++u) {
        const int t = time_of(u);
        const bool have_prev = u < T - 1;                    // forward-order predecessor = the step processed next
        uint32_t dyk[2][4];                                  // dY of units 8 j + 2 q, +1 (bf16 pair)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int j = 0; j < 4; ++j)
                dyk[h][j] = live[h] ? *reinterpret_cast<const uint32_t *>(a.dY + ((int64_t)t * B + row[h]) * 2 * H + dir * H + n0 + 8 * j + 2 * q) : 0u;
        float acc[16];
        if (u > 0) {
            if (u == 1 && !mbar_wait_bounded(wfull, 0, err)) atomicExch(err, 2u);
            uint64_t *pending = nullptr;
            for (int kb = 0; kb < nkb; ++kb, ++it) {
                const int s = it % STAGES;
                if (!mbar_wait_bounded(full + s, (it / STAGES) & 1, err)) atomicExch(err, 3u);
                if (kb < 16) MR_TRACE(u, 8 + kb);
                const uint32_t a_addr = smem_u32(As + s * kBwdATile), b_addr = smem_u32(Ws + kb * kBwdWTile);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < BK / WGMMA_K; ++k)
                    Wgmma<kBwdBN>::mma<0, 0>(acc, desc_kmajor(a_addr, k), desc_kmajor(b_addr, k), (kb | k) != 0);
                wgmma_commit();
                wgmma_wait<1>();                                 // the previous k-block has retired: its slot is free
                if (pending && leader) mbar_arrive(pending);
                pending = empty + s;
            }
            MR_TRACE(u, 2);
            wgmma_wait<0>();
            if (pending && leader) mbar_arrive(pending);
        } else {
#pragma unroll
            for (int k = 0; k < 16; ++k) acc[k] = 0.f;
        }
        MR_TRACE(u, 3);
        if (!mbar_wait_bounded(gfull, u & 1, err)) atomicExch(err, 6u);
        if (!mbar_wait_bounded(cfull + (u & 1), (u >> 1) & 1, err)) atomicExch(err, 7u);
        if (have_prev && !mbar_wait_bounded(cfull + ((u + 1) & 1), ((u + 1) >> 1) & 1, err)) atomicExch(err, 8u);
        const unsigned char *cc = Cs + (u & 1) * kBwdATile, *cp = Cs + ((u + 1) & 1) * kBwdATile;
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                // gates of units 8 j + 2 q, +1: one 16-byte chunk of gate box j / 2; c, c_prev: 8 bytes of chunk 2 j + q / 2
                const uint4 gk = *reinterpret_cast<const uint4 *>(Gs + (j >> 1) * kBwdATile + swz(rl[h], 4 * (j & 1) + q));
                const uint32_t coff = swz(rl[h], 2 * j + (q >> 1)) + 8 * (q & 1);
                const float2 c2 = *reinterpret_cast<const float2 *>(cc + coff);
                const float2 p2 = have_prev ? *reinterpret_cast<const float2 *>(cp + coff) : make_float2(0.f, 0.f);
                const __nv_bfloat162 *g2 = reinterpret_cast<const __nv_bfloat162 *>(&gk);
                const float2 dy = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&dyk[h][j]));
                const float cf[2] = {c2.x, c2.y}, cpf[2] = {p2.x, p2.y}, dyf[2] = {dy.x, dy.y};
                float dgf[8];
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const float2 fi = __bfloat1622float2(g2[2 * e]);
                    const float2 fg = __bfloat1622float2(g2[2 * e + 1]);
                    const LstmUnitGrad d = lstm_unit_bwd<CellFast>(fi.x, fi.y, fg.x, fg.y, cf[e], cpf[e],
                                                                   dyf[e] + acc[4 * j + 2 * h + e], dcs[h][2 * j + e]);
                    dgf[4 * e] = d.di;
                    dgf[4 * e + 1] = d.df;
                    dgf[4 * e + 2] = d.dg;
                    dgf[4 * e + 3] = d.do_;
                    dcs[h][2 * j + e] = d.dc_prev;
                }
                if (live[h])
                    *reinterpret_cast<uint4 *>(a.dG + ((int64_t)(dir * T + t) * B + row[h]) * 4 * H + 4 * (n0 + 8 * j + 2 * q)) =
                        make_uint4(pack_bf16x2(dgf[0], dgf[1]), pack_bf16x2(dgf[2], dgf[3]), pack_bf16x2(dgf[4], dgf[5]),
                                   pack_bf16x2(dgf[6], dgf[7]));
            }
        MR_TRACE(u, 4);
        named_bar_sync<kMmaThreads>(1);                      // dG_t stored; the gates and c_t tiles are read
        MR_TRACE(u, 5);
        if (leader) {
            MR_TRACE(u, 6);
            red_release_add(flag, 1u);
            MR_TRACE(u, 7);
            if (u + 1 < T) load_gates(u + 1);
            if (u + 2 < T) load_cell(u + 2);                 // into the buffer that held c_t of this step
        }
    }
    if (T == 1 && leader && !mbar_wait_bounded(wfull, 0, err)) atomicExch(err, 2u);   // no TMA load outlives the CTA
}

// 3-D tiled map over a row-major [outer, mid, inner] tensor, box {box_inner, box_mid, 1}, 128-byte swizzle
int make_map_3d(CUtensorMap *m, const void *base, CUtensorMapDataType dt, int esize, int64_t inner, int64_t mid, int64_t outer,
                int box_inner, int box_mid, bool swizzle = true) {
    EncodeTiledFn fn = encode_fn();
    if (!fn) { set_cuda_error(cudaErrorUnknown, "cuTensorMapEncodeTiled entry point"); return MR_ERR_CUDA; }
    cuuint64_t dims[3] = {(cuuint64_t)inner, (cuuint64_t)mid, (cuuint64_t)outer};
    cuuint64_t strides[2] = {(cuuint64_t)inner * esize, (cuuint64_t)mid * inner * esize};
    cuuint32_t box[3] = {(cuuint32_t)box_inner, (cuuint32_t)box_mid, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = fn(m, dt, 3, const_cast<void *>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    swizzle ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_cuda_error(cudaErrorInvalidValue, "cuTensorMapEncodeTiled(3d)"); return MR_ERR_CUDA; }
    return MR_OK;
}

int resident_ok(const void *kern, int threads, size_t smem, int ctas) {
    int dev = 0, sms = 0, per_sm = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 0;
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, threads, smem) != cudaSuccess) return 0;
    return ctas <= sms * per_sm;
}

constexpr int kBwdStages = 16;                // the whole 64 x 4H dG row block of a step at H = 256: no slot is refilled within a step
long long *g_trace = nullptr;

// flags: [dir][row tile] arrival counters for the finer (backward, 64-row) tiling, then the error word
int seq_flag_words(int B) { return 2 * ceil_div(B, kSeqRows) + 1; }

// A timed-out inter-CTA wait leaves garbage in the outputs and a non-zero error word.  Callers that never read the word
// (a training loop inside a CUDA graph) must still notice: if the word is set, the head of the output is overwritten with
// NaN, which reaches the loss (forward) or every weight gradient (backward) -- no host synchronisation needed.
__global__ void lstm_seq_poison_kernel(const unsigned *err, bf16 *out, int64_t n) {
    if (*err == 0u) return;
    const bf16 nan = __float2bfloat16(__int_as_float(0x7fc00000));
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) out[i] = nan;
}

// The persistent kernels spin on flags written by other CTAs of the same grid, so the WHOLE grid must be co-resident.
// A cooperative launch makes that a guarantee of the runtime (the grid is gang-scheduled, or the launch fails) instead
// of an occupancy estimate that concurrent work -- NCCL, the weight-gradient side stream -- could invalidate.
template <typename... Args>
cudaError_t launch_cooperative(void (*kern)(Args...), dim3 grid, int threads, size_t smem, cudaStream_t st, Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = dim3((unsigned)threads, 1, 1); cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeCooperative;
    at[0].val.cooperative = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kern, args...);
}

}  // namespace

extern "C" {

/* Development aid: clock64 stamps [T][32] of CTA (0,0,0) for the next launches (NULL = off).  Slots: 0 peers' arrival
 * seen, 1 TMA issued (producer); 2 last MMA committed, 3 accumulator in registers, 4 stores issued, 5 warpgroup barrier
 * passed, 6 release issued, 7 arrival posted (consumer warpgroup 0).  Backward only: 8 + kb k-block kb (< 16) arrived at
 * the MMA warpgroup, 20 + kb k-block kb (4..11) issued by the producer. */
int mr_lstm_seq_set_trace(void *buf) { g_trace = (long long *)buf; return MR_OK; }

/* Whole-sequence recurrence of one bidirectional LSTM layer, forward.  See include/megreader_b200.h. */
int mr_lstm_seq_fwd_tcgen05(const void *const *Whh, void *G, const float *const *bias, float *C, void *Y,
                            unsigned *flags, int T, int B, int H, void *stream) {
    if (T <= 0 || B <= 0 || H <= 0 || H % 64) return MR_ERR_UNSUPPORTED;
    if (!Whh || !Whh[0] || !Whh[1] || !G || !bias || !bias[0] || !bias[1] || !C || !Y || !flags) return MR_ERR_NULL_POINTER;
    if ((int64_t)2 * T * B >= (int64_t)1 << 31) return MR_ERR_UNSUPPORTED;
    const int nkb = H / BK, row_tiles = ceil_div(B, BM), words = seq_flag_words(B);
    const size_t smem = (size_t)nkb * (16384 + 8192) + 32768 + 8192 + 13 * 8 + 1024;
    if (nkb > 8 || smem > 227 * 1024) return MR_ERR_UNSUPPORTED;      /* afull[8]; in practice shared memory allows H <= 384 */
    auto kern = lstm_seq_fwd_kernel;
    { int rc_attr = ensure_dyn_smem((const void *)kern, smem, "lstm seq fwd smem attr"); if (rc_attr) return rc_attr; }
    dim3 grid((unsigned)row_tiles, (unsigned)(4 * H / kBN), 2);
    if (!resident_ok((const void *)kern, kFwdThreads, smem, (int)(grid.x * grid.y * grid.z))) return MR_ERR_UNSUPPORTED;
    CUtensorMap ty, tw[2];
    int rc = make_map(&ty, Y, 2 * H, (int64_t)T * B, 2 * H, BK, BM);
    if (rc) return rc;
    for (int d = 0; d < 2; ++d) {
        rc = make_map(&tw[d], Whh[d], H, 4 * H, H, BK, kBN);
        if (rc) return rc;
    }
    CUtensorMap tg3, tc3;
    rc = make_map_3d(&tg3, G, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, 4 * H, B, (int64_t)2 * T, BK, kSeqRows);
    if (rc) return rc;
    rc = make_map_3d(&tc3, C, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, H, B, (int64_t)2 * T, kBN / 4, kSeqRows, false);   // 64-byte rows: no swizzle
    if (rc) return rc;
    SeqFwdArgs a;
    a.G = (bf16 *)G; a.bias[0] = bias[0]; a.bias[1] = bias[1]; a.C = C; a.Y = (bf16 *)Y; a.flags = flags;
    a.err = flags + words - 1; a.trace = g_trace;
    a.T = T; a.B = B; a.H = H;
    MR_CUDA_TRY(cudaMemsetAsync(flags, 0, sizeof(unsigned) * words, (cudaStream_t)stream), "lstm seq flags");
    MR_CUDA_TRY(launch_cooperative(kern, grid, kFwdThreads, smem, (cudaStream_t)stream, ty, tw[0], tw[1], tg3, tc3, a), "lstm_seq_fwd_kernel");
    rc = check_launch("lstm_seq_fwd_kernel");
    if (rc) return rc;
    lstm_seq_poison_kernel<<<8, 256, 0, (cudaStream_t)stream>>>(flags + words - 1, (bf16 *)Y, (int64_t)T * B * 2 * H);
    return check_launch("lstm_seq_poison_kernel");
}

int mr_lstm_seq_bwd_tcgen05(const void *const *WhhT, const void *G, const float *C, const void *dY, void *dG,
                            unsigned *flags, int T, int B, int H, void *stream) {
    if (T <= 0 || B <= 0 || H <= 0 || H % 64) return MR_ERR_UNSUPPORTED;
    if (!WhhT || !WhhT[0] || !WhhT[1] || !G || !C || !dY || !dG || !flags) return MR_ERR_NULL_POINTER;
    if ((int64_t)2 * T * B >= (int64_t)1 << 31) return MR_ERR_UNSUPPORTED;
    const int nkb = 4 * H / BK, row_tiles = ceil_div(B, kSeqRows), words = seq_flag_words(B);
    const size_t smem = (size_t)(kBwdStages + 4) * kBwdATile + (size_t)nkb * kBwdWTile + (2 * kBwdStages + 4) * 8 + 1024;
    if (smem > 227 * 1024) return MR_ERR_UNSUPPORTED;
    auto kern = lstm_seq_bwd_kernel<kBwdStages>;
    { int rc_attr = ensure_dyn_smem((const void *)kern, smem, "lstm seq bwd smem attr"); if (rc_attr) return rc_attr; }
    dim3 grid((unsigned)row_tiles, (unsigned)(H / kBwdBN), 2);
    if (!resident_ok((const void *)kern, kBwdThreads, smem, (int)(grid.x * grid.y * grid.z))) return MR_ERR_UNSUPPORTED;
    CUtensorMap tdg, tw[2];
    int rc = make_map(&tdg, dG, 4 * H, (int64_t)2 * T * B, 4 * H, BK, kSeqRows);
    if (rc) return rc;
    for (int d = 0; d < 2; ++d) {
        rc = make_map(&tw[d], WhhT[d], 4 * H, H, 4 * H, BK, kBwdBN);      // W_hh^T [H, 4H]: K (= gate index) contiguous
        if (rc) return rc;
    }
    CUtensorMap tg3, tc3;
    rc = make_map_3d(&tg3, G, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, 4 * H, B, (int64_t)2 * T, BK, kSeqRows);
    if (rc) return rc;
    rc = make_map_3d(&tc3, C, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, H, B, (int64_t)2 * T, kBwdBN, kSeqRows);
    if (rc) return rc;
    SeqBwdArgs a;
    a.G = (const bf16 *)G; a.C = C; a.dY = (const bf16 *)dY; a.dG = (bf16 *)dG; a.flags = flags;
    a.err = flags + words - 1; a.trace = g_trace;
    a.T = T; a.B = B; a.H = H;
    MR_CUDA_TRY(cudaMemsetAsync(flags, 0, sizeof(unsigned) * words, (cudaStream_t)stream), "lstm seq flags");
    MR_CUDA_TRY(launch_cooperative(kern, grid, kBwdThreads, smem, (cudaStream_t)stream, tdg, tw[0], tw[1], tg3, tc3, a), "lstm_seq_bwd_kernel");
    rc = check_launch("lstm_seq_bwd_kernel");
    if (rc) return rc;
    lstm_seq_poison_kernel<<<8, 256, 0, (cudaStream_t)stream>>>(flags + words - 1, (bf16 *)dG, (int64_t)2 * T * B * 4 * H);
    return check_launch("lstm_seq_poison_kernel");
}

}  // extern "C"
