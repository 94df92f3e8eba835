// Persistent bidirectional-LSTM recurrence for sm_90a (decoders/crnn.py:13,17 nn.LSTM inside BidirectionalLSTM).
//
// The recurrence h_t = cell(Gx_t + h_{t-1} W_hh^T) is T dependent steps of a small GEMM ([B,H] x [H,4H]) plus a
// transcendental-heavy cell.  Launched step by step it is launch- and latency-bound (2 launches x T x 2 layers x
// fwd/bwd = 520 short launches in the CRNN train step).  Here ONE launch runs the whole sequence of one layer,
// both directions:
//   * the CTA grid tiles (batch rows / 128) x (gate columns / 64) x direction and stays resident for all T steps;
//   * each CTA keeps its W_hh slice in shared memory for the whole sequence (loaded once by TMA);
//   * per step, the h_{t-1} tile is TMA-loaded from the layer output Y itself (L2-resident), one MMA warpgroup (wgmma)
//     accumulates the recurrent product and publishes it as a shared-memory tile, 16 epilogue warps add the
//     x-projection, apply the cell and write h_t, c_t and the activated gates; the cell state (fwd) / its gradient (bwd) never leaves registers;
//   * the CTAs that share batch rows exchange h_t (fwd) / dG_t (bwd) through global memory and a monotonically
//     increasing arrival counter per (direction, row tile): writers  st -> bar.sync -> __threadfence -> atomicAdd,
//     readers  ld.acquire spin -> fence.proxy.async -> TMA.  All CTAs must be co-resident: the host refuses grids
//     larger than the device can hold (MR_ERR_UNSUPPORTED -> callers use the per-step kernels).
// Gate columns are UNIT-MAJOR (column 4*j + g = gate g of hidden unit j; g = i,f,g,o) as in gemm_tcgen05.cu.
// Every wait is bounded: on timeout the CTA records an error word (flags[2*row_tiles]) and runs to completion with
// undefined results instead of hanging the device.
#include "wgmma.cuh"
#include "lstm_cell.cuh"
#include <stdlib.h>

namespace {

constexpr int kBN = 64;                       // gate columns (fwd) / hidden units (bwd) per CTA
constexpr int kMma0 = 640;                    // producer warp, an idle warp, 16 epilogue warps, padded to a warpgroup boundary
constexpr int kThreads = kMma0 + kMmaThreads; // ... and the MMA warpgroup
constexpr int kEpiThreads = 16 * 32;

__device__ __forceinline__ uint32_t ld_acquire(const unsigned *p) {
    uint32_t v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }
__device__ __forceinline__ void epi_bar_sync() { asm volatile("bar.sync 1, %0;" ::"n"(kEpiThreads) : "memory"); }

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
__device__ __forceinline__ void tma_store_commit_wait() {
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}
// 16-byte chunk `c` of row `r` in a [rows x 128 B] tile written by TMA with the 128-byte swizzle (tile base 1024-aligned)
__device__ __forceinline__ uint32_t swz(int r, int c) { return (uint32_t)(r * 128 + ((c ^ (r & 7)) << 4)); }

struct SeqFwdArgs {
    bf16 *G;                  // [2, T, B, 4H] unit-major: x-projection on entry, activated gates on exit
    const float *bias[2];     // [4H] unit-major, b_ih + b_hh
    float *C;                 // [2, T, B, H] cell states (saved for the backward pass)
    bf16 *Y;                  // [T, B, 2H] layer output: direction d owns columns [d*H, (d+1)*H)
    unsigned *flags;          // [2 * row_tiles + 1], zeroed before launch; last word = error
    long long *trace;         // optional [T][8] clock64 stamps of CTA (0,0,0) (mr_lstm_seq_set_trace), else NULL
    int T, B, H;
};

__global__ void __launch_bounds__(kThreads, 1)
lstm_seq_fwd_kernel(const __grid_constant__ CUtensorMap tmY, const __grid_constant__ CUtensorMap tmW0,
                    const __grid_constant__ CUtensorMap tmW1, const __grid_constant__ CUtensorMap tmG3,
                    const __grid_constant__ CUtensorMap tmC3, SeqFwdArgs a) {
    extern __shared__ unsigned char smem_raw[];
    unsigned char *smem = (unsigned char *)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    const int nkb = a.H / BK;
    unsigned char *As = smem;                             // nkb x [128 rows x 128 B]   h_{t-1} tile, K-major SW128
    unsigned char *Ws = smem + nkb * 16384;               // nkb x [ 64 rows x 128 B]   W_hh slice, K-major SW128
    unsigned char *Gt = Ws + nkb * 8192;                  // 2 x [128 rows x 128 B]     gates tile: x-projection in, activations out
    unsigned char *Ct = Gt + 32768;                       // [128 rows x 64 B]          cell-state tile (16 units fp32), out
    float *acc_tile = (float *)(Ct + 8192);               // [128 rows x (64 + 1)] fp32      recurrent product of this step
    uint64_t *wfull = (uint64_t *)(Ct + 8192 + AccTile<kBN>::BYTES);
    uint64_t *afull = wfull + 1;                          // [8]
    uint64_t *acc_full = afull + 8;
    uint64_t *gfull = acc_full + 1;                       // [2]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int dir = blockIdx.z;
    const CUtensorMap *tmW = dir ? &tmW1 : &tmW0;
    const int m0 = blockIdx.x * BM, n0 = blockIdx.y * kBN;
    const int T = a.T, B = a.B, H = a.H;
    unsigned *flag = a.flags + dir * gridDim.x + blockIdx.x;
    unsigned *err = a.flags + 2 * gridDim.x;
    const uint32_t arrivals = gridDim.y;
    long long *trace = (blockIdx.x | blockIdx.y | blockIdx.z) == 0 ? a.trace : nullptr;

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&tmY);
        tma_prefetch_desc(tmW);
        tma_prefetch_desc(&tmG3);
        tma_prefetch_desc(&tmC3);
        mbar_init(wfull, 1);
        for (int i = 0; i < 8; ++i) mbar_init(afull + i, 1);
        mbar_init(acc_full, 1);
        mbar_init(gfull, 1);
        mbar_init(gfull + 1, 1);
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == 0) {
        if (elect_one()) {
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
    } else if (threadIdx.x >= kMma0) {
        const int mt = threadIdx.x - kMma0;
        if (mt != 0) trace = nullptr;
        AccTile<kBN> acc;
        if (!mbar_wait_bounded(wfull, 0, err)) atomicExch(err, 2u);
        for (int s = 1; s < T; ++s) {
            for (int kb = 0; kb < nkb; ++kb) {
                if (!mbar_wait_bounded(afull + kb, (s - 1) & 1, err)) atomicExch(err, 3u);
                const uint32_t a_addr = smem_u32(As + kb * 16384), b_addr = smem_u32(Ws + kb * 8192);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < BK / WGMMA_K; ++k)
                    acc.mma<0, 0>(desc_kmajor(a_addr, k), desc_kmajor(a_addr, k, 1), desc_kmajor(b_addr, k), (kb | k) != 0);
                wgmma_commit();
            }
            wgmma_wait<0>();
            // the epilogue warps drained the previous step's tile before any peer could post the arrival this step waited for
            acc.store(acc_tile, mt);
            mma_group_sync();
            if (mt == 0) { mbar_arrive(acc_full); MR_TRACE(s, 2); }
        }
    } else if (warp >= 2 && threadIdx.x < 64 + kEpiThreads) {
        if (threadIdx.x != 64) trace = nullptr;
        const int qd = warp & 3, grp = (warp - 2) >> 2;        // 32-row quarter of the tile, group of 16 gate columns = 4 units
        const int row = m0 + qd * 32 + lane;
        const int col0 = n0 + grp * 16, j0 = col0 >> 2;
        const bool live = row < B;
        float bb[16];
#pragma unroll
        for (int v = 0; v < 4; ++v) {
            const float4 b4 = __ldg(reinterpret_cast<const float4 *>((dir ? a.bias[1] : a.bias[0]) + col0) + v);
            bb[4 * v] = b4.x; bb[4 * v + 1] = b4.y; bb[4 * v + 2] = b4.z; bb[4 * v + 3] = b4.w;
        }
        float cst[4] = {0.f, 0.f, 0.f, 0.f};
        // The gates tile [128 rows x 64 columns] of every step comes and goes by TMA (row-per-thread global accesses
        // cost 32 wavefronts per warp instruction): loaded two steps ahead into a double
        // buffer, activated in place, stored together with the cell-state tile by the leader thread.
        const bool leader = threadIdx.x == 64;
        const int rl = qd * 32 + lane;
        auto time_of = [&](int s) { return dir ? T - 1 - s : s; };
        auto load_gates = [&](int s) {
            mbar_expect_tx(gfull + (s & 1), 16384);
            tma_load_3d(&tmG3, gfull + (s & 1), Gt + (s & 1) * 16384, n0, m0, dir * T + time_of(s));
        };
        if (leader) {
            load_gates(0);
            if (T > 1) load_gates(1);
        }
        for (int s = 0; s < T; ++s) {
            const int t = time_of(s);
            unsigned char *gt = Gt + (s & 1) * 16384;
            if (!mbar_wait_bounded(gfull + (s & 1), (s >> 1) & 1, err)) atomicExch(err, 6u);
            uint4 pk[2];
            pk[0] = *reinterpret_cast<const uint4 *>(gt + swz(rl, 2 * grp));
            pk[1] = *reinterpret_cast<const uint4 *>(gt + swz(rl, 2 * grp + 1));
            uint32_t r[16];
            if (s > 0) {
                if (!mbar_wait_bounded(acc_full, (s - 1) & 1, err)) atomicExch(err, 4u);
                acc_ld<16>(acc_tile, AccTile<kBN>::LD, qd * 32, grp * 16, r);
            } else {
#pragma unroll
                for (int j = 0; j < 16; ++j) r[j] = 0;
            }
            MR_TRACE(s, 3);
            float act[16];
#pragma unroll
            for (int j = 0; j < 16; ++j) act[j] = 0.f;
            if (live) {
                float pre[16];
#pragma unroll
                for (int v = 0; v < 2; ++v) {
                    const __nv_bfloat162 *h2 = reinterpret_cast<const __nv_bfloat162 *>(&pk[v]);
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        const float2 f = __bfloat1622float2(h2[e]);
                        pre[v * 8 + 2 * e] = f.x;
                        pre[v * 8 + 2 * e + 1] = f.y;
                    }
                }
                float hn[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const LstmUnit c = lstm_unit_fwd<CellFast>(
                        pre[4 * u] + __uint_as_float(r[4 * u]) + bb[4 * u], pre[4 * u + 1] + __uint_as_float(r[4 * u + 1]) + bb[4 * u + 1],
                        pre[4 * u + 2] + __uint_as_float(r[4 * u + 2]) + bb[4 * u + 2], pre[4 * u + 3] + __uint_as_float(r[4 * u + 3]) + bb[4 * u + 3],
                        cst[u]);
                    cst[u] = c.c;
                    hn[u] = c.h;
                    act[4 * u] = c.i; act[4 * u + 1] = c.f; act[4 * u + 2] = c.g; act[4 * u + 3] = c.o;
                }
                uint2 hp;
                __nv_bfloat162 *hh = reinterpret_cast<__nv_bfloat162 *>(&hp);
                hh[0] = __floats2bfloat162_rn(hn[0], hn[1]);
                hh[1] = __floats2bfloat162_rn(hn[2], hn[3]);
                *reinterpret_cast<uint2 *>(a.Y + ((int64_t)t * B + row) * 2 * H + dir * H + j0) = hp;
            }
            // h_t is all the peers wait for: post the arrival before the state that only the backward pass reads
            MR_TRACE(s, 4);
            epi_bar_sync();                                      // every h_t of this tile stored, accumulator drained
            MR_TRACE(s, 5);
            if (threadIdx.x == 64) {
                __threadfence();
                MR_TRACE(s, 6);
                atomicAdd(flag, 1u);
                MR_TRACE(s, 7);
            }
            // activated gates back into the tile, cell state into its tile (rows >= B are clipped by the TMA store)
#pragma unroll
            for (int v = 0; v < 2; ++v) {
                uint4 o4;
                __nv_bfloat162 *h2 = reinterpret_cast<__nv_bfloat162 *>(&o4);
#pragma unroll
                for (int e = 0; e < 4; ++e) h2[e] = __floats2bfloat162_rn(act[v * 8 + 2 * e], act[v * 8 + 2 * e + 1]);
                *reinterpret_cast<uint4 *>(gt + swz(rl, 2 * grp + v)) = o4;
            }
            *reinterpret_cast<float4 *>(Ct + rl * 64 + grp * 16) = make_float4(cst[0], cst[1], cst[2], cst[3]);     // plain rows
            fence_proxy_async();                                 // generic-proxy tile writes -> visible to the TMA stores
            epi_bar_sync();
            if (leader) {
                const int z = dir * T + t;
                tma_store_3d(&tmG3, gt, n0, m0, z);
                tma_store_3d(&tmC3, Ct, n0 >> 2, m0, z);
                tma_store_commit_wait_read();                    // both tiles may be overwritten again
                if (s + 2 < T) load_gates(s + 2);
            }
        }
    }
}

struct SeqBwdArgs {
    const bf16 *G;            // [2, T, B, 4H] activated gates (unit-major) from the forward pass
    const float *C;           // [2, T, B, H]
    const bf16 *dY;           // [T, B, 2H] gradient of the layer output
    bf16 *dG;                 // [2, T, B, 4H] gate gradients, out (unit-major)
    unsigned *flags;
    long long *trace;
    int T, B, H;
};

// Backward recurrence: dh_{t} += dG_{t_next} W_hh needs the FULL gate-gradient row block [128 x 4H] per output tile, so
// the per-step operand traffic is (H / units-per-CTA) x the dG tile.  32 hidden units per CTA spread the step over
// (B/128) x (H/32) x 2 CTAs (64 at the CRNN shape).  A thread owns one batch row, so direct global access
// would touch 32 different rows per warp instruction.
// Instead the per-step operands -- activated gates [128 x 128] bf16 and cell state [128 x 32] fp32 -- are TMA-loaded as
// swizzled tiles one step ahead and read conflict-free from shared memory; the gate gradients are written back into the
// gates tile and leave through one TMA store.  c_prev of this step is the c tile of the next one: one new tile per step.
constexpr int kBwdBN = 32;
constexpr int kBwdWTile = kBwdBN * 128;       // one k-block of W_hh^T: 32 unit rows x 128 B (K-major, SW128)

template <int STAGES>
__global__ void __launch_bounds__(kThreads, 1)
lstm_seq_bwd_kernel(const __grid_constant__ CUtensorMap tmDG, const __grid_constant__ CUtensorMap tmW0,
                    const __grid_constant__ CUtensorMap tmW1, const __grid_constant__ CUtensorMap tmG3,
                    const __grid_constant__ CUtensorMap tmDG3, const __grid_constant__ CUtensorMap tmC3, SeqBwdArgs a) {
    extern __shared__ unsigned char smem_raw[];
    unsigned char *smem = (unsigned char *)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    const int nkb = 4 * a.H / BK;
    unsigned char *As = smem;                             // STAGES x [128 rows x 128 B]  dG_{next} k-block, K-major SW128
    unsigned char *Gs = smem + STAGES * 16384;            // 2 x [128 x 128 B]            gates of this step -> dG of this step
    unsigned char *Cs = Gs + 32768;                       // 2 x [128 x 128 B]            cell-state tiles (fp32, 32 units)
    unsigned char *Ws = Cs + 32768;                       // nkb x [32 rows x 128 B]      W_hh^T[n0.., kb*64..), K-major SW128
    float *acc_tile = (float *)(Ws + nkb * kBwdWTile);    // [128 rows x (32 + 1)] fp32    recurrent product of this step
    uint64_t *wfull = (uint64_t *)(Ws + nkb * kBwdWTile + AccTile<kBwdBN>::BYTES);
    uint64_t *full = wfull + 1;
    uint64_t *empty = full + STAGES;
    uint64_t *acc_full = empty + STAGES;
    uint64_t *gfull = acc_full + 1;
    uint64_t *cfull = gfull + 1;                          // [2]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int dir = blockIdx.z;
    const CUtensorMap *tmW = dir ? &tmW1 : &tmW0;
    const int m0 = blockIdx.x * BM, n0 = blockIdx.y * kBwdBN;
    const int T = a.T, B = a.B, H = a.H;
    unsigned *flag = a.flags + dir * gridDim.x + blockIdx.x;
    unsigned *err = a.flags + 2 * gridDim.x;
    const uint32_t arrivals = gridDim.y;
    long long *trace = (blockIdx.x | blockIdx.y | blockIdx.z) == 0 ? a.trace : nullptr;

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&tmDG);
        tma_prefetch_desc(tmW);
        tma_prefetch_desc(&tmG3);
        tma_prefetch_desc(&tmDG3);
        tma_prefetch_desc(&tmC3);
        mbar_init(wfull, 1);
        for (int i = 0; i < STAGES; ++i) { mbar_init(full + i, 1); mbar_init(empty + i, 1); }
        mbar_init(acc_full, 1);
        mbar_init(gfull, 1);
        mbar_init(cfull, 1);
        mbar_init(cfull + 1, 1);
        fence_barrier_init();
    }
    __syncthreads();

    // processing order u = 0..T-1 is the reverse of the forward order: direction 0 walks t = T-1..0, direction 1 t = 0..T-1
    if (warp == 0) {
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
                    mbar_expect_tx(full + s, 16384);
                    if (kb >= 4 && kb < 12) MR_TRACE(u, 20 + kb);
                    tma_load_2d(&tmDG, full + s, As + s * 16384, kb * BK, (dir * T + t_next) * B + m0);
                }
                MR_TRACE(u, 1);
            }
        }
    } else if (threadIdx.x >= kMma0) {
        const int mt = threadIdx.x - kMma0;
        if (mt != 0) trace = nullptr;
        AccTile<kBwdBN> acc;
        if (!mbar_wait_bounded(wfull, 0, err)) atomicExch(err, 2u);
        int it = 0;
        for (int u = 1; u < T; ++u) {
            uint64_t *pending = nullptr;
            for (int kb = 0; kb < nkb; ++kb, ++it) {
                const int s = it % STAGES;
                if (!mbar_wait_bounded(full + s, (it / STAGES) & 1, err)) atomicExch(err, 3u);
                if (kb < 16) MR_TRACE(u, 8 + kb);
                const uint32_t a_addr = smem_u32(As + s * 16384), b_addr = smem_u32(Ws + kb * kBwdWTile);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < BK / WGMMA_K; ++k)
                    acc.mma<0, 0>(desc_kmajor(a_addr, k), desc_kmajor(a_addr, k, 1), desc_kmajor(b_addr, k), (kb | k) != 0);
                wgmma_commit();
                wgmma_wait<1>();                                 // the previous k-block has retired: its slot is free
                if (pending && mt == 0) mbar_arrive(pending);
                pending = empty + s;
            }
            wgmma_wait<0>();
            if (pending && mt == 0) mbar_arrive(pending);
            acc.store(acc_tile, mt);
            mma_group_sync();
            if (mt == 0) { mbar_arrive(acc_full); MR_TRACE(u, 2); }
        }
    } else if (warp >= 2 && threadIdx.x < 64 + kEpiThreads) {
        const bool leader = threadIdx.x == 64;
        if (!leader) trace = nullptr;
        const int qd = warp & 3, grp = (warp - 2) >> 2;        // 32-row quarter of the tile, group of 8 hidden units
        const int rl = qd * 32 + lane, row = m0 + rl;
        const int j0 = n0 + grp * 8;
        const bool live = row < B;
        // this thread's slices of the staged tiles: gates/dG 4 chunks in box (grp >> 1), cell state 2 chunks
        unsigned char *gtile = Gs + (grp >> 1) * 16384;
        const int gch = (grp & 1) * 4, cch = grp * 2;
        float dcs[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) dcs[j] = 0.f;
        auto time_of = [&](int u) { return dir ? u : T - 1 - u; };
        auto load_gates = [&](int u) {
            const int z = dir * T + time_of(u);
            mbar_expect_tx(gfull, 32768);
            tma_load_3d(&tmG3, gfull, Gs, 4 * n0, m0, z);
            tma_load_3d(&tmG3, gfull, Gs + 16384, 4 * n0 + 64, m0, z);
        };
        auto load_cell = [&](int u) {
            mbar_expect_tx(cfull + (u & 1), 16384);
            tma_load_3d(&tmC3, cfull + (u & 1), Cs + (u & 1) * 16384, n0, m0, dir * T + time_of(u));
        };
        if (leader) {
            load_gates(0);
            load_cell(0);
            if (T > 1) load_cell(1);
        }
        for (int u = 0; u < T; ++u) {
            const int t = time_of(u);
            const bool have_prev = u < T - 1;                    // forward-order predecessor = the step processed next
            uint4 dyk = make_uint4(0, 0, 0, 0);
            if (live)
                dyk = *reinterpret_cast<const uint4 *>(a.dY + ((int64_t)t * B + row) * 2 * H + dir * H + j0);
            if (!mbar_wait_bounded(gfull, u & 1, err)) atomicExch(err, 6u);
            if (!mbar_wait_bounded(cfull + (u & 1), (u >> 1) & 1, err)) atomicExch(err, 7u);
            if (have_prev && !mbar_wait_bounded(cfull + ((u + 1) & 1), ((u + 1) >> 1) & 1, err)) atomicExch(err, 8u);
            uint4 gk[4];
            float4 c4[2], p4[2];
#pragma unroll
            for (int e = 0; e < 4; ++e) gk[e] = *reinterpret_cast<const uint4 *>(gtile + swz(rl, gch + e));
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                c4[e] = *reinterpret_cast<const float4 *>(Cs + (u & 1) * 16384 + swz(rl, cch + e));
                p4[e] = have_prev ? *reinterpret_cast<const float4 *>(Cs + ((u + 1) & 1) * 16384 + swz(rl, cch + e))
                                  : make_float4(0.f, 0.f, 0.f, 0.f);
            }
            uint32_t r[8];
            if (u > 0) {
                if (!mbar_wait_bounded(acc_full, (u - 1) & 1, err)) atomicExch(err, 4u);
                acc_ld<8>(acc_tile, AccTile<kBwdBN>::LD, qd * 32, grp * 8, r);
            } else {
#pragma unroll
                for (int j = 0; j < 8; ++j) r[j] = 0;
            }
            MR_TRACE(u, 3);
            {
                const __nv_bfloat162 *dy2 = reinterpret_cast<const __nv_bfloat162 *>(&dyk);
                float dyf[8];
#pragma unroll
                for (int e = 0; e < 4; ++e) { const float2 f = __bfloat1622float2(dy2[e]); dyf[2 * e] = f.x; dyf[2 * e + 1] = f.y; }
                const float cf[8] = {c4[0].x, c4[0].y, c4[0].z, c4[0].w, c4[1].x, c4[1].y, c4[1].z, c4[1].w};
                const float cpf[8] = {p4[0].x, p4[0].y, p4[0].z, p4[0].w, p4[1].x, p4[1].y, p4[1].z, p4[1].w};
#pragma unroll
                for (int h = 0; h < 4; ++h) {                    // 2 units (8 gate values) per 16-byte chunk
                    const __nv_bfloat162 *g2 = reinterpret_cast<const __nv_bfloat162 *>(&gk[h]);
                    float dgf[8];
#pragma unroll
                    for (int w2 = 0; w2 < 2; ++w2) {
                        const int uu = h * 2 + w2;
                        const float2 fi = __bfloat1622float2(g2[2 * w2]);
                        const float2 fg = __bfloat1622float2(g2[2 * w2 + 1]);
                        const LstmUnitGrad d = lstm_unit_bwd<CellFast>(fi.x, fi.y, fg.x, fg.y, cf[uu], cpf[uu],
                                                                       dyf[uu] + __uint_as_float(r[uu]), dcs[uu]);
                        dgf[w2 * 4] = d.di;
                        dgf[w2 * 4 + 1] = d.df;
                        dgf[w2 * 4 + 2] = d.dg;
                        dgf[w2 * 4 + 3] = d.do_;
                        dcs[uu] = d.dc_prev;
                    }
                    uint4 o4;
                    __nv_bfloat162 *p2 = reinterpret_cast<__nv_bfloat162 *>(&o4);
#pragma unroll
                    for (int e = 0; e < 4; ++e) p2[e] = __floats2bfloat162_rn(dgf[2 * e], dgf[2 * e + 1]);
                    *reinterpret_cast<uint4 *>(gtile + swz(rl, gch + h)) = o4;       // rows >= B are clipped by the TMA store
                }
            }
            fence_proxy_async();                                 // generic-proxy tile writes -> visible to the TMA store
            MR_TRACE(u, 4);
            epi_bar_sync();
            MR_TRACE(u, 5);
            if (leader) {
                const int z = dir * T + t;
                tma_store_3d(&tmDG3, Gs, 4 * n0, m0, z);
                tma_store_3d(&tmDG3, Gs + 16384, 4 * n0 + 64, m0, z);
                tma_store_commit_wait();                         // gate gradients written (and the tile is free again)
                fence_proxy_async_global();
                __threadfence();
                MR_TRACE(u, 6);
                atomicAdd(flag, 1u);
                MR_TRACE(u, 7);
                if (u + 1 < T) load_gates(u + 1);
                if (u + 2 < T) load_cell(u + 2);                 // into the buffer that held c_t of this step
            }
        }
    }
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

constexpr int kBwdStages = 5;
long long *g_trace = nullptr;

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
 * seen, 1 TMA issued, 2 last MMA committed, 3 accumulator in registers, 4 stores issued, 5 tile barrier passed,
 * 6 __threadfence done, 7 arrival posted. */
int mr_lstm_seq_set_trace(void *buf) { g_trace = (long long *)buf; return MR_OK; }

/* Whole-sequence recurrence of one bidirectional LSTM layer, forward.  See include/megreader_b200.h. */
int mr_lstm_seq_fwd_tcgen05(const void *const *Whh, void *G, const float *const *bias, float *C, void *Y,
                            unsigned *flags, int T, int B, int H, void *stream) {
    if (T <= 0 || B <= 0 || H <= 0 || H % 64) return MR_ERR_UNSUPPORTED;
    if (!Whh || !Whh[0] || !Whh[1] || !G || !bias || !bias[0] || !bias[1] || !C || !Y || !flags) return MR_ERR_NULL_POINTER;
    if ((int64_t)2 * T * B >= (int64_t)1 << 31) return MR_ERR_UNSUPPORTED;
    const int nkb = H / BK, row_tiles = ceil_div(B, BM);
    const size_t smem = (size_t)nkb * (16384 + 8192) + 32768 + 8192 + AccTile<kBN>::BYTES + 16 * 8 + 1024;
    if (nkb > 8 || smem > 227 * 1024) return MR_ERR_UNSUPPORTED;      /* afull[8]; in practice shared memory allows H <= 384 */
    auto kern = lstm_seq_fwd_kernel;
    { int rc_attr = ensure_dyn_smem((const void *)kern, smem, "lstm seq fwd smem attr"); if (rc_attr) return rc_attr; }
    dim3 grid((unsigned)row_tiles, (unsigned)(4 * H / kBN), 2);
    if (!resident_ok((const void *)kern, kThreads, smem, (int)(grid.x * grid.y * grid.z))) return MR_ERR_UNSUPPORTED;
    CUtensorMap ty, tw[2];
    int rc = make_map(&ty, Y, 2 * H, (int64_t)T * B, 2 * H, BK, BM);
    if (rc) return rc;
    for (int d = 0; d < 2; ++d) {
        rc = make_map(&tw[d], Whh[d], H, 4 * H, H, BK, kBN);
        if (rc) return rc;
    }
    CUtensorMap tg3, tc3;
    rc = make_map_3d(&tg3, G, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, 4 * H, B, (int64_t)2 * T, BK, BM);
    if (rc) return rc;
    rc = make_map_3d(&tc3, C, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, H, B, (int64_t)2 * T, kBN / 4, BM, false);   // 64-byte rows: no swizzle
    if (rc) return rc;
    SeqFwdArgs a;
    a.G = (bf16 *)G; a.bias[0] = bias[0]; a.bias[1] = bias[1]; a.C = C; a.Y = (bf16 *)Y; a.flags = flags; a.trace = g_trace;
    a.T = T; a.B = B; a.H = H;
    MR_CUDA_TRY(cudaMemsetAsync(flags, 0, sizeof(unsigned) * (2 * row_tiles + 1), (cudaStream_t)stream), "lstm seq flags");
    MR_CUDA_TRY(launch_cooperative(kern, grid, kThreads, smem, (cudaStream_t)stream, ty, tw[0], tw[1], tg3, tc3, a), "lstm_seq_fwd_kernel");
    rc = check_launch("lstm_seq_fwd_kernel");
    if (rc) return rc;
    lstm_seq_poison_kernel<<<8, 256, 0, (cudaStream_t)stream>>>(flags + 2 * row_tiles, (bf16 *)Y, (int64_t)T * B * 2 * H);
    return check_launch("lstm_seq_poison_kernel");
}

int mr_lstm_seq_bwd_tcgen05(const void *const *WhhT, const void *G, const float *C, const void *dY, void *dG,
                            unsigned *flags, int T, int B, int H, void *stream) {
    if (T <= 0 || B <= 0 || H <= 0 || H % 64) return MR_ERR_UNSUPPORTED;
    if (!WhhT || !WhhT[0] || !WhhT[1] || !G || !C || !dY || !dG || !flags) return MR_ERR_NULL_POINTER;
    if ((int64_t)2 * T * B >= (int64_t)1 << 31) return MR_ERR_UNSUPPORTED;
    const int nkb = 4 * H / BK, row_tiles = ceil_div(B, BM);
    const size_t smem = (size_t)kBwdStages * 16384 + 65536 + (size_t)nkb * kBwdWTile + AccTile<kBwdBN>::BYTES + (2 * kBwdStages + 8) * 8 + 1024;
    if (smem > 227 * 1024) return MR_ERR_UNSUPPORTED;
    auto kern = lstm_seq_bwd_kernel<kBwdStages>;
    { int rc_attr = ensure_dyn_smem((const void *)kern, smem, "lstm seq bwd smem attr"); if (rc_attr) return rc_attr; }
    dim3 grid((unsigned)row_tiles, (unsigned)(H / kBwdBN), 2);
    if (!resident_ok((const void *)kern, kThreads, smem, (int)(grid.x * grid.y * grid.z))) return MR_ERR_UNSUPPORTED;
    CUtensorMap tdg, tw[2];
    int rc = make_map(&tdg, dG, 4 * H, (int64_t)2 * T * B, 4 * H, BK, BM);
    if (rc) return rc;
    for (int d = 0; d < 2; ++d) {
        rc = make_map(&tw[d], WhhT[d], 4 * H, H, 4 * H, BK, kBwdBN);      // W_hh^T [H, 4H]: K (= gate index) contiguous
        if (rc) return rc;
    }
    CUtensorMap tg3, tdg3, tc3;
    rc = make_map_3d(&tg3, G, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, 4 * H, B, (int64_t)2 * T, BK, BM);
    if (rc) return rc;
    rc = make_map_3d(&tdg3, dG, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, 4 * H, B, (int64_t)2 * T, BK, BM);
    if (rc) return rc;
    rc = make_map_3d(&tc3, C, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, H, B, (int64_t)2 * T, kBwdBN, BM);
    if (rc) return rc;
    SeqBwdArgs a;
    a.G = (const bf16 *)G; a.C = C; a.dY = (const bf16 *)dY; a.dG = (bf16 *)dG; a.flags = flags; a.trace = g_trace;
    a.T = T; a.B = B; a.H = H;
    MR_CUDA_TRY(cudaMemsetAsync(flags, 0, sizeof(unsigned) * (2 * row_tiles + 1), (cudaStream_t)stream), "lstm seq flags");
    MR_CUDA_TRY(launch_cooperative(kern, grid, kThreads, smem, (cudaStream_t)stream, tdg, tw[0], tw[1], tg3, tdg3, tc3, a), "lstm_seq_bwd_kernel");
    rc = check_launch("lstm_seq_bwd_kernel");
    if (rc) return rc;
    lstm_seq_poison_kernel<<<8, 256, 0, (cudaStream_t)stream>>>(flags + 2 * row_tiles, (bf16 *)dG, (int64_t)2 * T * B * 4 * H);
    return check_launch("lstm_seq_poison_kernel");
}

}  // extern "C"
